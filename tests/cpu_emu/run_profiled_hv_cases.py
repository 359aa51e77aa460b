"""python -m tests.cpu_emu.run_profiled_hv_cases <libhv_profiled_kernel_emu.so> [n_cases]: the profiled forms of the emulated ring
kernel (hv_ring_profiled_kernel, ifb_hv_kernel.cuh) against the oracle chain: tests/profile_oracle.apply_plan of to_bgra(source), then
tests/orient_oracle.gather, then oracle.scale_and_render.  Matrix and gray plans; flags 1..8; BGRA, RGBA32 and RGB24 sources, RGB24
at every byte phase mod 16; ring depths 4 and 6; three and four channels; both simple store epilogues; sharpen; strips and bands.
Also the body of the AddressSanitizer run (the test starts it in a subprocess with libasan preloaded)."""
import ctypes as C
import sys

import numpy as np

import imageflow_b200 as ifb
import oracle
from tests import cpu_emu, orient_oracle, profile_oracle as pf, util
from tests.cpu_emu.run_oriented_hv_cases import JF_FLIP_X, JF_FLIP_Y, ORIENT, HV_ORI_TRANSPOSE
from tests.cpu_emu.run_rows_hv_cases import HV_SRC_RGB24, HV_SRC_RGBA, to_bgra

HV_SRC_BGRA, PF_MATRIX, PF_GRAY = 0, 1, 2
ALL = (1, 2, 3, 4, 5, 6, 7, 8)
P3 = "display_p3_v4"
# (source format, stored in_w, in_h, out_w, out_h, filter, flags, profile, kwargs of run_profiled)
CASES = [
    ("rgb24", 480, 352, 96, 80, 2, ALL, P3, dict(n_bands=3)),                       # ring depth 4, three channels, bands
    ("rgba", 480, 352, 96, 80, 2, ALL, P3, dict(alpha=True, n_bands=2)),            # four channels
    ("bgra", 480, 352, 96, 80, 2, ALL, "adobe_rgb_v2", dict()),                     # BGRA frames
    ("rgb24", 480, 352, 96, 80, 2, ALL, "gray22_v2", dict(phase=5)),                # a gray plan
    ("bgra", 480, 352, 96, 80, 2, (1, 3, 6), "gray22_v2", dict(alpha=True)),
    ("rgb24", 540, 400, 96, 72, 6, (1, 3, 6, 8), P3, dict(n_bands=2, phase=3)),     # Lanczos3: ring depth 6, three channels
    ("rgba", 540, 400, 96, 72, 6, (1, 2, 5, 7), P3, dict(alpha=True)),              # ring depth 6, four channels
    ("bgra", 540, 400, 96, 72, 6, (1, 4, 6), "adobe_rgb_v2", dict(linear=False)),   # sRGB space
    ("rgb24", 1280, 96, 24, 320, 2, (5, 8), P3, dict(strip_cols=16, phase=11)),     # many strips
    ("rgb24", 512, 384, 96, 128, 13, (1, 2, 6), P3, dict(sharpen=50.0, n_bands=2, linear=False)),   # CatmullRom, sharpen
    ("rgba", 332, 277, 61, 79, 2, (1, 3, 7), "gray22_v2", dict(alpha=True, content="cutout")),      # cut-out alpha
] + [("rgb24", 101, 70, 23, 17, 2, (1, 2, 7) if p % 2 else (3, 6, 8), P3, dict(phase=p)) for p in range(16)]   # every byte phase


def profile(name):
    kind, data = pf.fixtures()[name]
    return ifb.SourceProfile.icc(data) if kind == "icc" else ifb.SourceProfile.icc_gray(data)


class ProfDev(C.Structure):                              # imageflow_b200/csrc/ifb_profile_step.cuh
    _fields_ = [("trc", (C.c_float * 256) * 3), ("m", C.c_float * 9), ("gray", C.c_uint8 * 256)]


def run_profiled(lib, src, fmt, plan, canvas, flag, *, x=0, y=0, w=None, h=None, filter=2, sharpen=0.0, linear=True, alpha_meaningful=False,
                 grid=1, strip_cols=64, n_bands=1, sb_low16=0x400, phase=0):
    """One launch of the emulated profiled ring kernel for the resample of orient(transform(to_bgra(src), plan), flag), with the plan
    behind the job array; otherwise as run_rows_oriented_hv_cases.run_hv_rows_oriented.  Returns the result canvas."""
    form, fx, fy = ORIENT[flag] if flag != 1 else (0, False, False)
    ih, iw, bpp = src.shape
    phase = phase if fmt == "rgb24" else 0
    oiw, oih = (ih, iw) if form == HV_ORI_TRANSPOSE else (iw, ih)
    w = canvas.shape[1] - x if w is None else w
    h = canvas.shape[0] - y if h is None else h
    info, blob = cpu_emu.hv_plan(ifb, oiw, oih, w, h, filter, sharpen, strip_cols, n_bands, alpha_meaningful)
    assert blob is not None, ("not a ring geometry", iw, ih, w, h)
    t_lin, t_srgb, lut = cpu_emu.transfer_tables(ifb)
    assert lib.emu_sizeof_profdev() == C.sizeof(ProfDev)
    row_bytes = phase + iw * bpp
    pitch = (row_bytes + 15) // 16 * 16
    mem = np.zeros((ih - 1) * pitch + row_bytes, np.uint8)              # no byte after the last row's: AddressSanitizer sees an overrun
    assert mem.ctypes.data % 16 == 0
    for j in range(ih):
        mem[j * pitch + phase:j * pitch + row_bytes] = src[j].reshape(-1)
    out = np.ascontiguousarray(canvas.copy())
    buf = (C.c_uint8 * (C.sizeof(cpu_emu.JobDev) + C.sizeof(ProfDev)))()
    j = cpu_emu.JobDev.from_buffer(buf)
    j.in_ = mem.ctypes.data + phase; j.out = out.ctypes.data + y * out.strides[0] + x * 4
    j.in_stride, j.out_stride, j.in_xoff = pitch, out.strides[0], phase
    cpu_emu.set_job_store(j, t_lin, t_srgb, linear=linear, alpha_meaningful=alpha_meaningful, compose=0, matte=(0, 0, 0, 0), color_matrix=None)
    j.flags |= (JF_FLIP_X if fx else 0) | (JF_FLIP_Y if fy else 0)
    pd = ProfDev.from_buffer(buf, C.sizeof(cpu_emu.JobDev))
    C.memmove(pd.trc, np.ascontiguousarray(plan.trc, np.float32).ctypes.data, 3 * 256 * 4)
    C.memmove(pd.m, np.ascontiguousarray(plan.m, np.float32).ctypes.data, 9 * 4)
    C.memmove(pd.gray, np.ascontiguousarray(plan.gray, np.uint8).ctypes.data, 256)
    in_ptrs = (C.c_void_p * 1)(mem.ctypes.data)
    in_whs = np.array([row_bytes if fmt == "rgb24" else iw, ih, pitch], np.uint32)
    offs = np.array([info.o_strips, info.o_hw, info.o_hdone, info.o_vw, info.o_vdone, info.o_bands, info.total], np.uint64)
    dims = np.array([oiw, oih, w, h, info.cap_px], np.uint32)
    src_kind = {"bgra": HV_SRC_BGRA, "rgba": HV_SRC_RGBA, "rgb24": HV_SRC_RGB24}[fmt]
    bad = lib.emu_hv_launch_profiled(info.av, 4 if alpha_meaningful else 3, 1 if linear else 2, form, src_kind, plan.kind, grid,
                                     C.cast(buf, C.c_void_p), 1, C.cast(in_ptrs, C.c_void_p), in_whs.ctypes.data, t_lin.ctypes.data,
                                     t_srgb.ctypes.data, lut.ctypes.data, blob.ctypes.data, offs.ctypes.data, dims.ctypes.data,
                                     info.n_strips, info.n_bands, sb_low16)
    assert bad == 0, f"{bad} bad shared-memory accesses / box origins / barrier states (or no such form)"
    return out, info


def load(so):
    L = C.CDLL(so)
    L.emu_sizeof_profdev.restype = C.c_uint32
    L.emu_hv_launch_profiled.restype = C.c_int
    L.emu_hv_launch_profiled.argtypes = [C.c_int] * 6 + [C.c_uint, C.c_void_p, C.c_uint32] + [C.c_void_p] * 8 + [C.c_int, C.c_int, C.c_uint32]
    return L


def run(so, limit=None):
    """every (case, flag) bit-exact; returns the number of (case, flag) runs and the (ring depth, channels, source, plan) forms reached"""
    L = load(so)
    lut = cpu_emu.transfer_tables(ifb)[2]
    n, reached = 0, set()
    for (fmt, iw, ih, ow, oh, flt, flags, pname, kw) in CASES:
        kw = dict(kw)
        alpha = kw.pop("alpha", False) or fmt == "rgba"
        common = dict(filter=flt, alpha_meaningful=alpha, linear=kw.pop("linear", True), sharpen=kw.pop("sharpen", 0.0))
        if kw.pop("content", "noise") == "cutout":
            bgra = synth_cutout(iw, ih)
        else:
            bgra = util.noise(iw, ih, seed=iw + oh, alpha_mode="mixed")
        canvas = util.noise(ow + 5, oh + 3, seed=3, alpha_mode="mixed")
        rows = np.ascontiguousarray(bgra[..., [2, 1, 0, 3]])
        src = {"bgra": bgra, "rgba": rows, "rgb24": np.ascontiguousarray(rows[..., :3])}[fmt]
        as_bgra = bgra if fmt == "bgra" else to_bgra(src)
        plan = ifb.source_profile_plan(profile(pname))
        srgb = pf.apply_plan(plan, lut, as_bgra)
        for flag in flags:
            exp = canvas.copy()
            oracle.scale_and_render(np.ascontiguousarray(orient_oracle.gather(srgb, flag)), exp, x=2, y=1, w=ow, h=oh, **common)
            got, info = run_profiled(L, src, fmt, plan, canvas, flag, x=2, y=1, w=ow, h=oh, **common, **kw)
            d = np.abs(got.astype(np.int16) - exp.astype(np.int16))
            assert d.max() == 0, (fmt, iw, ih, ow, oh, flt, flag, pname, kw, int(d.max()), int((d > 0).sum()))
            reached.add((info.av, 4 if alpha else 3, fmt, plan.kind))
            n += 1
            if limit and n >= limit:
                return n, reached
    return n, reached


def synth_cutout(iw, ih):
    from imageflow_b200 import synth
    return synth.cutout_np(iw, ih, seed=iw + ih)


if __name__ == "__main__":
    n, reached = run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else None)
    print("profiled cases bit-exact:", n, "forms:", len(reached))
