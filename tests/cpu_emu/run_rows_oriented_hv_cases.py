"""python -m tests.cpu_emu.run_rows_oriented_hv_cases <libhv_rows_oriented_kernel_emu.so> [n_cases]: the oriented row-format forms of the
emulated hv_ring_kernel (ifb_hv_kernel.cuh, ORI = HV_ORI_FLIP / HV_ORI_TRANSPOSE, SRC = HV_SRC_RGBA / HV_SRC_RGB24) against the
oracle's resample of the rows converted to BGRA and oriented in numpy.
Also the body of the AddressSanitizer run (the test starts it in a subprocess with libasan preloaded)."""
import ctypes as C
import sys

import numpy as np

import imageflow_b200 as ifb
import oracle
from imageflow_b200 import synth
from tests import cpu_emu, orient_oracle, util
from tests.cpu_emu.run_oriented_hv_cases import JF_FLIP_X, JF_FLIP_Y, ORIENT, HV_ORI_TRANSPOSE
from tests.cpu_emu.run_rows_hv_cases import HV_SRC_RGB24, HV_SRC_RGBA, to_bgra

ALL = (2, 3, 4, 5, 6, 7, 8)
# (bytes per pixel, stored in_w, in_h, out_w, out_h, filter, flags, kwargs of run_hv_rows_oriented); out_w x out_h is the size on the canvas
CASES = [
    (3, 960, 540, 128, 128, 2, ALL, dict(n_bands=3)),                                # config-2 ratios, every flag, bands
    (4, 960, 540, 128, 128, 2, ALL, dict(alpha=True, n_bands=2)),                    # RGBA32, four channels
    (3, 962, 541, 128, 128, 2, ALL, dict(phase=7)),                                  # widths not a multiple of four, odd byte phase
    (3, 540, 960, 96, 170, 6, (3, 6, 8), dict(alpha=True, n_bands=2, phase=5)),      # Lanczos3: ring depth 6, four channels (alpha 255)
    (4, 540, 960, 96, 170, 6, (2, 5, 7), dict(alpha=True, n_bands=2)),
    (3, 960, 540, 128, 128, 6, (4, 7), dict(linear=False, phase=13)),                # ring depth 6, three channels, sRGB space
    (4, 960, 540, 128, 128, 6, (3, 6), dict(linear=False)),
    (3, 800, 600, 300, 400, 2, (2, 6, 7), dict(alpha=True, compose=1, cm="sepia", phase=2)),   # composite over the canvas, colour matrix
    (4, 800, 600, 300, 400, 2, (4, 8), dict(alpha=True, compose=1, cm="sepia")),
    (3, 1280, 96, 24, 320, 2, (5, 8), dict(strip_cols=16, alpha=True, compose=2, phase=11)),   # many strips, matte
    (4, 96, 1280, 320, 24, 2, (5, 7), dict(strip_cols=16, alpha=True, compose=2)),
    (3, 260, 250, 59, 61, 2, ALL, dict(n_bands=4, phase=9)),                         # ragged sizes, short bands
    (3, 33, 17, 5, 7, 2, ALL, dict(alpha=True, phase=15)),                           # smaller than one TMA box
    (4, 12, 9, 5, 4, 2, (2, 3, 6, 8), dict(alpha=True)),
    (3, 400, 300, 75, 100, 4, (3, 6), dict(alpha=True, linear=False, strip_cols=16, phase=3)),   # Ginseng (ring depth 6), sRGB space
    (4, 640, 480, 150, 200, 2, (3, 6, 8), dict(content="cutout", alpha=True, compose=1)),      # cut-out content: the store's alpha branches
    (4, 640, 480, 150, 200, 2, (2, 7), dict(content="cutout", alpha=True, compose=2, linear=False, cm="sepia")),
    (3, 512, 384, 96, 128, 13, (2, 5, 6), dict(sharpen=50.0, n_bands=2, phase=4)),  # CatmullRom, sharpen
    (4, 512, 384, 96, 128, 13, (4, 7), dict(sharpen=50.0, alpha=True)),
    (3, 333, 277, 61, 79, 2, (2, 3, 7, 8), dict(alpha=True, n_bands=5, phase=1)),    # odd widths, reversed source x
] + [(3, 101, 70, 23, 17, 2, (2, 7) if p % 2 else (3, 6, 8), dict(phase=p, alpha=p % 2 == 1)) for p in range(16)]   # every byte phase mod 16


def ring_eligible(bpp, iw, flag):
    """whether the engine runs the job on the ring kernel (enqueue_locked): RGBA32 keeps the BGRA rule (source x reversed needs a
    stored width that is a multiple of four); RGB24 has no width rule"""
    return bpp == 3 or not (ORIENT[flag][1] and iw % 4)


def ring_form_exists(bpp, av, alpha, linear, compose, cm, flag):
    """whether the engine compiled this ring form (HvEntry::rows_ori): the RGB24 flip forms at ring depth 6 with three channels and
    the general or the linear store epilogue would spill; they are not compiled and their jobs take the generic pair"""
    simple_srgb = compose == 0 and cm is None and not linear
    return not (bpp == 3 and av == 6 and not alpha and ORIENT[flag][0] != HV_ORI_TRANSPOSE and not simple_srgb)


def run_hv_rows_oriented(lib, rows, canvas, flag, *, x=0, y=0, w=None, h=None, filter=2, sharpen=0.0, linear=True, alpha_meaningful=False,
                         compose=0, matte=(0, 0, 0, 0), color_matrix=None, grid=1, strip_cols=64, n_bands=1, sb_low16=0x400, phase=0):
    """One launch of the emulated oriented row-format ring kernel for the resample of orient(to_bgra(rows), flag): the plan tables of
    the ORIENTED geometry; the stored rows `phase` bytes past a 16-byte aligned base (RGB24; RGBA32 rows are 16-byte aligned as the
    engine requires), rows a multiple of 16 bytes apart, in a buffer that ends with the last row's last byte; the TMA descriptor,
    in_xoff and flags as enqueue_locked / tmap_for / make_job set them.  Returns the result canvas, or None if the geometry is not a
    ring geometry."""
    form, fx, fy = ORIENT[flag]
    ih, iw, bpp = rows.shape
    phase = phase if bpp == 3 else 0
    oiw, oih = (ih, iw) if form == HV_ORI_TRANSPOSE else (iw, ih)
    w = canvas.shape[1] - x if w is None else w
    h = canvas.shape[0] - y if h is None else h
    info, blob = cpu_emu.hv_plan(ifb, oiw, oih, w, h, filter, sharpen, strip_cols, n_bands, alpha_meaningful)
    if blob is None:
        return None
    t_lin, t_srgb, lut = cpu_emu.transfer_tables(ifb)
    assert lib.emu_hv_sizeof_jobdev() == C.sizeof(cpu_emu.JobDev)
    row_bytes = phase + iw * bpp
    pitch = (row_bytes + 15) // 16 * 16
    mem = np.zeros((ih - 1) * pitch + row_bytes, np.uint8)              # no byte after the last row's: AddressSanitizer sees an overrun
    assert mem.ctypes.data % 16 == 0
    for j in range(ih):
        mem[j * pitch + phase:j * pitch + row_bytes] = rows[j].reshape(-1)
    out = np.ascontiguousarray(canvas.copy())
    jobs = (cpu_emu.JobDev * 1)()
    j = jobs[0]
    j.in_ = mem.ctypes.data + phase; j.out = out.ctypes.data + y * out.strides[0] + x * 4
    j.in_stride, j.out_stride, j.in_xoff = pitch, out.strides[0], phase
    cpu_emu.set_job_store(j, t_lin, t_srgb, linear=linear, alpha_meaningful=alpha_meaningful, compose=compose, matte=matte, color_matrix=color_matrix)
    j.flags |= (JF_FLIP_X if fx else 0) | (JF_FLIP_Y if fy else 0)
    in_ptrs = (C.c_void_p * 1)(mem.ctypes.data)
    in_whs = np.array([row_bytes if bpp == 3 else iw, ih, pitch], np.uint32)
    offs = np.array([info.o_strips, info.o_hw, info.o_hdone, info.o_vw, info.o_vdone, info.o_bands, info.total], np.uint64)
    dims = np.array([oiw, oih, w, h, info.cap_px], np.uint32)
    simple = compose == 0 and color_matrix is None
    bad = lib.emu_hv_launch_rows_oriented(info.av, 4 if alpha_meaningful else 3, int(simple), form, HV_SRC_RGB24 if bpp == 3 else HV_SRC_RGBA,
                                          grid, C.cast(jobs, C.c_void_p), 1, C.cast(in_ptrs, C.c_void_p), in_whs.ctypes.data,
                                          t_lin.ctypes.data, t_srgb.ctypes.data, lut.ctypes.data, blob.ctypes.data, offs.ctypes.data,
                                          dims.ctypes.data, info.n_strips, info.n_bands, sb_low16)
    assert bad == 0, f"{bad} bad shared-memory accesses / box origins / barrier states"
    return out


def load(so):
    L = C.CDLL(so)
    L.emu_hv_sizeof_jobdev.restype = C.c_uint32
    L.emu_hv_launch_rows_oriented.restype = C.c_int
    L.emu_hv_launch_rows_oriented.argtypes = [C.c_int] * 5 + [C.c_uint, C.c_void_p, C.c_uint32] + [C.c_void_p] * 8 + [C.c_int, C.c_int, C.c_uint32]
    return L


def run(so, limit=None):
    """every (case, flag) bit-exact; returns the number of (case, flag) runs"""
    L = load(so)
    n = 0
    for (bpp, iw, ih, ow, oh, flt, flags, kw) in CASES:
        kw = dict(kw)
        alpha = kw.pop("alpha", False)
        cm = ifb.color_filter_matrix(0) if kw.pop("cm", None) == "sepia" else None
        common = dict(filter=flt, alpha_meaningful=alpha, linear=kw.pop("linear", True), compose=kw.pop("compose", 0), matte=(40, 120, 250, 200),
                      color_matrix=cm, sharpen=kw.pop("sharpen", 0.0))
        if kw.pop("content", "noise") == "cutout":
            bgra, canvas = synth.cutout_np(iw, ih, seed=iw + oh), synth.cutout_canvas_np(ow + 5, oh + 3, seed=3)
        else:
            bgra = util.noise(iw, ih, seed=iw + oh + bpp, alpha_mode="mixed")
            canvas = util.noise(ow + 5, oh + 3, seed=3, alpha_mode="mixed")
        rows = np.ascontiguousarray(bgra[..., [2, 1, 0, 3]][..., :bpp])        # decoder rows: R, G, B(, A)
        for flag in flags:
            if not ring_eligible(bpp, iw, flag):
                continue
            oiw, oih = (ih, iw) if ORIENT[flag][0] == HV_ORI_TRANSPOSE else (iw, ih)
            info, _ = cpu_emu.hv_plan(ifb, oiw, oih, ow, oh, flt, common["sharpen"], kw.get("strip_cols", 64), 1, alpha)
            assert info.ok, ("not a ring geometry", iw, ih, ow, oh, flt, flag)
            if not ring_form_exists(bpp, info.av, alpha, common["linear"], common["compose"], cm, flag):
                continue
            exp = canvas.copy()
            oracle.scale_and_render(np.ascontiguousarray(orient_oracle.gather(to_bgra(rows), flag)), exp, x=2, y=1, w=ow, h=oh, **common)
            got = run_hv_rows_oriented(L, rows, canvas, flag, x=2, y=1, w=ow, h=oh, **common, **kw)
            assert got is not None, ("not a ring geometry", iw, ih, ow, oh, flt, flag)
            d = np.abs(got.astype(np.int16) - exp.astype(np.int16))
            assert d.max() == 0, (bpp, iw, ih, ow, oh, flt, flag, alpha, kw, int(d.max()), int((d > 0).sum()))
            n += 1
            if limit and n >= limit:
                return n
    return n


if __name__ == "__main__":
    print("oriented rows cases bit-exact:", run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else None))
