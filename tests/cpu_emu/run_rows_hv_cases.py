"""python -m tests.cpu_emu.run_rows_hv_cases <libhv_rows_kernel_emu.so> [n_cases]: the row-format forms of the emulated hv_ring_kernel
(ifb_hv_kernel.cuh, SRC = HV_SRC_RGBA / HV_SRC_RGB24) against the oracle's resample of the rows converted to BGRA in numpy.
Also the body of the AddressSanitizer run (the test starts it in a subprocess with libasan preloaded)."""
import ctypes as C
import sys

import numpy as np

import imageflow_b200 as ifb
import oracle
from imageflow_b200 import synth
from tests import cpu_emu, util

HV_SRC_RGBA, HV_SRC_RGB24 = 1, 2

# (bytes per pixel, in_w, in_h, out_w, out_h, filter, kwargs of run_hv_rows); out_w x out_h is the size on the canvas
CASES = [
    (3, 960, 540, 128, 128, 2, dict(n_bands=3)),                                     # config-2 ratios, 3 in_w a multiple of 16, bands
    (3, 962, 540, 128, 128, 2, dict(phase=7)),                                       # 3 in_w not a multiple of 16, odd byte phase
    (4, 960, 540, 128, 128, 2, dict(alpha=True, n_bands=2)),                         # RGBA32, four channels
    (3, 540, 960, 96, 170, 6, dict(alpha=True, n_bands=2, phase=5)),                 # Lanczos3: ring depth 6, four channels (alpha 255)
    (3, 960, 540, 128, 128, 6, dict(linear=False, phase=13)),                        # ring depth 6, three channels, sRGB space
    (4, 960, 540, 128, 128, 6, dict(linear=False)),
    (4, 800, 600, 300, 400, 2, dict(alpha=True, compose=1, cm="sepia")),             # composite over the canvas, colour matrix
    (3, 800, 600, 300, 400, 2, dict(compose=1, cm="sepia", phase=2)),
    (3, 96, 1280, 24, 320, 2, dict(strip_cols=16, alpha=True, compose=2, phase=11)),   # many strips, matte
    (4, 1280, 96, 320, 24, 2, dict(strip_cols=16, alpha=True, compose=2)),
    (3, 260, 250, 59, 61, 2, dict(n_bands=4, phase=9)),                              # ragged sizes, short bands
    (3, 33, 17, 5, 7, 2, dict(alpha=True, phase=15)),                                # smaller than one TMA box
    (4, 13, 9, 5, 4, 2, dict(alpha=True)),
    (3, 400, 300, 75, 100, 4, dict(alpha=True, linear=False, strip_cols=16, phase=3)),   # Ginseng (ring depth 6), sRGB space
    (4, 640, 480, 150, 200, 2, dict(content="cutout", alpha=True, compose=1)),       # cut-out content: the store's alpha branches
    (4, 640, 480, 150, 200, 2, dict(content="cutout", alpha=True, compose=2, linear=False, cm="sepia")),
    (3, 512, 384, 96, 128, 13, dict(sharpen=50.0, n_bands=2, phase=4)),              # CatmullRom, sharpen
    (4, 512, 384, 96, 128, 13, dict(sharpen=50.0, alpha=True)),
] + [(3, 101, 70, 23, 17, 2, dict(phase=p, alpha=p % 2 == 1)) for p in range(16)]      # every byte phase mod 16


def ring_form_exists(bpp, av, alpha, compose, cm):
    """whether the engine has this ring form (enqueue_locked): RGB24 with the general store epilogue at ring depth 6 and three
    channels is not compiled (it would spill) and takes the generic pair"""
    return not (bpp == 3 and av == 6 and not alpha and (compose != 0 or cm is not None))


def to_bgra(rows):
    """ifb200_pixel_convert_desc's RGB24_TO_BGRA / RGBA_TO_BGRA with opaque = 0, in numpy"""
    h, w, c = rows.shape
    out = np.full((h, w, 4), 255, np.uint8)
    out[..., 0], out[..., 1], out[..., 2] = rows[..., 2], rows[..., 1], rows[..., 0]
    if c == 4:
        out[..., 3] = rows[..., 3]
    return out


def run_hv_rows(lib, rows, canvas, *, x=0, y=0, w=None, h=None, filter=2, sharpen=0.0, linear=True, alpha_meaningful=False, compose=0,
                matte=(0, 0, 0, 0), color_matrix=None, grid=1, strip_cols=64, n_bands=1, sb_low16=0x400, phase=0):
    """One launch of the emulated row-format ring kernel for the resample of to_bgra(rows): the rows `phase` bytes past a 16-byte
    aligned base (RGB24; RGBA32 rows are 16-byte aligned as the engine requires), rows a multiple of 16 bytes apart, in a buffer that
    ends with the last row's last byte; the TMA descriptor, in_xoff and flags as enqueue_locked / tmap_for / make_job set them.
    Returns the result canvas, or None if the geometry is not a ring geometry."""
    ih, iw, bpp = rows.shape
    assert bpp == 4 or phase == 0 or bpp == 3
    phase = phase if bpp == 3 else 0
    w = canvas.shape[1] - x if w is None else w
    h = canvas.shape[0] - y if h is None else h
    info, blob = cpu_emu.hv_plan(ifb, iw, ih, w, h, filter, sharpen, strip_cols, n_bands, alpha_meaningful)
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
    in_ptrs = (C.c_void_p * 1)(mem.ctypes.data)
    in_whs = np.array([row_bytes if bpp == 3 else iw, ih, pitch], np.uint32)
    offs = np.array([info.o_strips, info.o_hw, info.o_hdone, info.o_vw, info.o_vdone, info.o_bands, info.total], np.uint64)
    dims = np.array([iw, ih, w, h, info.cap_px], np.uint32)
    simple = compose == 0 and color_matrix is None
    bad = lib.emu_hv_launch_rows(info.av, 4 if alpha_meaningful else 3, int(simple), HV_SRC_RGB24 if bpp == 3 else HV_SRC_RGBA, grid,
                                 C.cast(jobs, C.c_void_p), 1, C.cast(in_ptrs, C.c_void_p), in_whs.ctypes.data, t_lin.ctypes.data,
                                 t_srgb.ctypes.data, lut.ctypes.data, blob.ctypes.data, offs.ctypes.data, dims.ctypes.data, info.n_strips,
                                 info.n_bands, sb_low16)
    assert bad == 0, f"{bad} bad shared-memory accesses / box origins / barrier states"
    return out


def load(so):
    L = C.CDLL(so)
    L.emu_hv_sizeof_jobdev.restype = C.c_uint32
    L.emu_hv_launch_rows.restype = C.c_int
    L.emu_hv_launch_rows.argtypes = [C.c_int] * 4 + [C.c_uint, C.c_void_p, C.c_uint32] + [C.c_void_p] * 8 + [C.c_int, C.c_int, C.c_uint32]
    return L


def run(so, limit=None):
    """every case bit-exact; returns the number of cases run"""
    L = load(so)
    n = 0
    for (bpp, iw, ih, ow, oh, flt, kw) in CASES:
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
        info, _ = cpu_emu.hv_plan(ifb, iw, ih, ow, oh, flt, common["sharpen"], kw.get("strip_cols", 64), 1, alpha)
        assert info.ok, ("not a ring geometry", iw, ih, ow, oh, flt)
        if not ring_form_exists(bpp, info.av, alpha, common["compose"], cm):
            continue
        exp = canvas.copy()
        oracle.scale_and_render(to_bgra(rows), exp, x=2, y=1, w=ow, h=oh, **common)
        got = run_hv_rows(L, rows, canvas, x=2, y=1, w=ow, h=oh, **common, **kw)
        assert got is not None, ("not a ring geometry", iw, ih, ow, oh, flt)
        d = np.abs(got.astype(np.int16) - exp.astype(np.int16))
        assert d.max() == 0, (bpp, iw, ih, ow, oh, flt, alpha, kw, int(d.max()), int((d > 0).sum()))
        n += 1
        if limit and n >= limit:
            return n
    return n


if __name__ == "__main__":
    print("rows cases bit-exact:", run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else None))
