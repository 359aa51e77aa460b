"""CPU emulation of product CUDA kernels (test infrastructure): the kernel sources are compiled with g++ under an emulation of
the CUDA built-ins they use and run on small cases, so that indexing, arithmetic and -- under AddressSanitizer -- memory accesses
of a kernel can be checked without a GPU.  Nothing in the product imports this package."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "imageflow_b200", "csrc")
u32, f32 = C.c_uint32, C.c_float
# every emulator library is built with the same flags: the kernels' arithmetic is never contracted into fused multiply-adds it
# does not spell out (-ffp-contract=off), and the threaded emulators need std::barrier and std::thread (C++20, -pthread)
CXXFLAGS = ["-O1", "-g", "-std=c++20", "-pthread", "-shared", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unknown-pragmas",
            "-Wno-implicit-fallthrough"]
ASAN_FLAGS = ["-fsanitize=address", "-fno-omit-frame-pointer"]


def _libasan() -> str:
    """the path of g++'s libasan; skips the calling test when there is none (an instrumented build could not link)"""
    import pytest
    asan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan) or not os.path.exists(asan):
        pytest.skip("libasan not available")
    return asan


def build(out_dir: str, emu_source: str, *product_sources: str, sanitize: bool = False) -> str:
    """g++ of tests/cpu_emu/<emu_source> with the product's host sources imageflow_b200/csrc/<product_sources> it links, into a
    library in out_dir (instrumented by AddressSanitizer when `sanitize`).  Returns its path."""
    if sanitize:
        _libasan()
    name = os.path.splitext(emu_source)[0] + ("_asan" if sanitize else "")
    so = os.path.join(out_dir, f"lib{name}.so")
    cmd = ["g++", *CXXFLAGS, *(ASAN_FLAGS if sanitize else []), "-o", so, os.path.join(HERE, emu_source)]
    subprocess.run(cmd + [os.path.join(CSRC, s) for s in product_sources], check=True)
    return so


def run_under_asan(module: str, so: str, n: int, timeout: int = 1200) -> subprocess.CompletedProcess:
    """python -m tests.cpu_emu.<module> <so> <n> with libasan preloaded (the test is skipped when g++ has no libasan)"""
    env = dict(os.environ, LD_PRELOAD=_libasan(), ASAN_OPTIONS="detect_leaks=0:verify_asan_link_order=0", PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, "-m", f"tests.cpu_emu.{module}", so, str(n)], capture_output=True, text=True, cwd=ROOT,
                          env=env, timeout=timeout)


class JobDev(C.Structure):                          # imageflow_b200/csrc/ifb_types.cuh
    _fields_ = [("in_", C.c_void_p), ("out", C.c_void_p), ("in_stride", u32), ("out_stride", u32), ("flags", u32), ("in_xoff", u32),
                ("matte", f32 * 4), ("cm", f32 * 20)]


def transfer_tables(ifb):
    """(t_lin, t_srgb, lut16k): the library's byte-to-float tables of both working spaces and its linear-to-sRGB table"""
    t_lin, t_srgb, lut = np.zeros(256, np.float32), np.zeros(256, np.float32), np.zeros(16384, np.uint8)
    f32p, u8p = C.POINTER(C.c_float), C.POINTER(C.c_uint8)
    ifb.lib().ifb200_byte_to_float_table(1, t_lin.ctypes.data_as(f32p)); ifb.lib().ifb200_byte_to_float_table(0, t_srgb.ctypes.data_as(f32p))
    ifb.lib().ifb200_linear_to_srgb_table(lut.ctypes.data_as(u8p))
    return t_lin, t_srgb, lut


def set_job_store(j, t_lin, t_srgb, *, linear, alpha_meaningful, compose, matte, color_matrix):
    """JobDev's flags, premultiplied matte and transposed colour matrix, as make_job (ifb_engine.cu) sets them"""
    j.flags = (1 if linear else 0) | (2 if alpha_meaningful else 0) | (compose << 2)
    if compose == 2 and alpha_meaningful:
        T = t_lin if linear else t_srgb
        ma = np.float32(matte[3]) * np.float32(1.0 / 255.0)
        for c in range(3):
            j.matte[c] = float(np.float32(T[matte[c]]) * ma)
        j.matte[3] = float(ma)
    if color_matrix is not None:
        m = np.ascontiguousarray(color_matrix, np.float32).reshape(25)
        j.flags |= 16
        for c in range(4):
            for k in range(4):
                j.cm[c * 5 + k] = float(m[k * 5 + c])
            j.cm[c * 5 + 4] = float(np.float32(m[20 + c]) * np.float32(255.0))
        cm = np.array(list(j.cm), np.float32)
        if all(cm[15 + k] == (1.0 if k == 3 else 0.0) for k in range(5)) and all(cm[c * 5 + 3] == 0 and cm[c * 5 + 4] == 0 for c in range(3)):
            j.flags |= 32


def csr(ws):
    left = np.array([w[0] for w in ws], np.uint32); right = np.array([w[1] for w in ws], np.uint32)
    off = np.zeros(len(ws), np.uint32); off[1:] = np.cumsum([len(w[2]) for w in ws])[:-1]
    return left, right, off, np.concatenate([np.asarray(w[2], np.float32) for w in ws])


def run_tile2(lib, ifb, inp, canvas, *, x=0, y=0, w=None, h=None, filter=14, linear=True, alpha_meaningful=False, compose=0,
              matte=(0, 0, 0, 0), color_matrix=None, grid=3, jobs_repeat=1):
    """One launch of the emulated fused_tile2_kernel for `jobs_repeat` identical jobs (each on its own copy of the canvas);
    mirrors what enqueue_locked / make_job / build_tile do on the host (ifb_engine.cu).  Returns the list of result canvases."""
    L = lib
    ih, iw = inp.shape[:2]
    w = canvas.shape[1] - x if w is None else w
    h = canvas.shape[0] - y if h is None else h
    wv, wh = ifb.populate_weights(filter, h, ih), ifb.populate_weights(filter, w, iw)
    vl, vr, vo, vw = csr(wv); hl, hr, ho, hw = csr(wh)
    th = L.emu_tile2_tile_h()
    tiles_x, tiles_y = (w + 63) // 64, (h + th - 1) // th
    max_ic = max(int(hr[min(tx * 64 + 64, w) - 1]) - int(hl[tx * 64]) + 1 for tx in range(tiles_x))
    max_ir = max(int(vr[min(ty * th + th, h) - 1]) - int(vl[ty * th]) + 1 for ty in range(tiles_y))
    # the padded windows of the register forms, as build_tile() lays them out (ifb_engine.cu)
    span = 6
    t_vw = np.zeros((tiles_y * th, 8), np.float32); t_vq = np.zeros(tiles_y * th // 4, np.uint32)
    for ty in range(tiles_y):
        ya, yb = ty * th, min(ty * th + th, h)
        r0, r1 = int(vl[ya]), int(vr[yb - 1])
        for yq in range(ya, yb, 4):
            b0 = min(int(vl[yq]), max(r1 - min(r1, span - 1), r0))
            rows = range(yq, min(yq + 4, yb))
            fit = r1 - r0 + 1 >= span and all(int(vl[yy]) >= b0 and int(vr[yy]) < b0 + span for yy in rows)
            t_vq[yq // 4] = b0 + 1 if fit else 0
            if fit:
                for yy in rows:
                    for j in range(int(vl[yy]), int(vr[yy]) + 1):
                        t_vw[yy, j - b0] = vw[int(vo[yy]) + j - int(vl[yy])]
    h4 = int(max(int(r) - int(l) + 1 for l, r in zip(hl, hr)) <= 4)
    t_hw = np.zeros((tiles_x * 64, 4), np.float32)
    if h4:
        for xx in range(w):
            for j in range(int(hl[xx]), int(hr[xx]) + 1):
                t_hw[xx, j - int(hl[xx])] = hw[int(ho[xx]) + j - int(hl[xx])]
    plan = np.array([iw, ih, w, h, 64, th, tiles_x, tiles_y, max_ic, max_ir, h4], np.int32)
    t_lin, t_srgb, lut = transfer_tables(ifb)
    assert L.emu_tile2_sizeof_jobdev() == C.sizeof(JobDev)
    inp = np.ascontiguousarray(inp)
    outs = [np.ascontiguousarray(canvas.copy()) for _ in range(jobs_repeat)]
    jobs = (JobDev * jobs_repeat)()
    ch = 4 if alpha_meaningful else 3
    for j, o in zip(jobs, outs):
        j.in_ = inp.ctypes.data; j.out = o.ctypes.data + y * o.strides[0] + x * 4
        j.in_stride, j.out_stride = inp.strides[0], o.strides[0]
        set_job_store(j, t_lin, t_srgb, linear=linear, alpha_meaningful=alpha_meaningful, compose=compose, matte=matte, color_matrix=color_matrix)
    p = lambda a, t: a.ctypes.data_as(C.POINTER(t))
    rc = L.emu_tile2_launch(ch, int(linear), compose, int(color_matrix is not None), grid, C.cast(jobs, C.c_void_p), jobs_repeat,
                            p(t_lin, C.c_float), p(t_srgb, C.c_float), p(lut, C.c_uint8),
                            p(vl, u32), p(vr, u32), p(vo, u32), p(vw, C.c_float), p(hl, u32), p(hr, u32), p(ho, u32), p(hw, C.c_float),
                            p(plan, C.c_int32), p(t_vw, C.c_float), p(t_vq, u32), p(t_hw, C.c_float))
    assert rc == 0
    return outs


def load_tile2(so):
    L = C.CDLL(so)
    L.emu_tile2_sizeof_jobdev.restype = u32
    L.emu_tile2_tile_h.restype = C.c_int
    L.emu_tile2_launch.restype = C.c_int
    L.emu_tile2_launch.argtypes = [C.c_int] * 4 + [C.c_uint, C.c_void_p, u32] + [C.c_void_p] * 11 + [C.c_void_p] * 4
    return L


# ---------------------------------------------------------------------------------------------- hv_ring_kernel (ifb_hv_kernel.cuh)
class HvPlanInfo(C.Structure):                      # include/ifb200.h ifb200_hv_plan_info
    _fields_ = [("ok", C.c_int32), ("av", C.c_int32), ("n_strips", C.c_int32), ("n_bands", C.c_int32), ("cap_px", C.c_int32), ("avp", C.c_int32),
                ("o_strips", C.c_uint64), ("o_hw", C.c_uint64), ("o_hdone", C.c_uint64), ("o_vw", C.c_uint64), ("o_vdone", C.c_uint64),
                ("o_bands", C.c_uint64), ("total", C.c_uint64)]


def load_hv(so):
    L = C.CDLL(so)
    L.emu_hv_sizeof_jobdev.restype = u32
    L.emu_hv_launch.restype = C.c_int
    L.emu_hv_launch.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint, C.c_void_p, u32] + [C.c_void_p] * 8 + [C.c_int, C.c_int, u32]
    return L


def hv_plan(ifb, iw, ih, ow, oh, filter, sharpen=0.0, strip_cols=64, n_bands=1, alpha=False):
    """(info, blob) of ifb200_hv_plan_tables, or (info, None) when the geometry is not a ring-kernel geometry"""
    from imageflow_b200._lib import ResampleDesc
    L = ifb.lib()
    L.ifb200_hv_plan_tables.restype = C.c_int
    L.ifb200_hv_plan_tables.argtypes = [C.POINTER(ResampleDesc), C.c_int, C.c_int, C.POINTER(HvPlanInfo), C.c_void_p, C.c_size_t, C.c_char_p, C.c_size_t]
    d = ResampleDesc(); d.in_w, d.in_h, d.w, d.h, d.filter, d.sharpen_percent, d.alpha_meaningful = iw, ih, ow, oh, filter, sharpen, int(alpha)
    info = HvPlanInfo(); err = C.create_string_buffer(256)
    rc = L.ifb200_hv_plan_tables(C.byref(d), strip_cols, n_bands, C.byref(info), None, 0, err, 256)
    assert rc == 0, err.value
    if not info.ok:
        return info, None
    blob = np.zeros(int(info.total), np.uint8)
    rc = L.ifb200_hv_plan_tables(C.byref(d), strip_cols, n_bands, C.byref(info), blob.ctypes.data, blob.nbytes, err, 256)
    assert rc == 0, err.value
    return info, blob


def run_hv(lib, ifb, inp, canvas, *, x=0, y=0, w=None, h=None, filter=2, sharpen=0.0, linear=True, alpha_meaningful=False, compose=0,
           matte=(0, 0, 0, 0), color_matrix=None, grid=1, jobs_repeat=1, strip_cols=64, n_bands=1, sb_low16=0x400, in_xoff=0):
    """One launch of the emulated hv_ring_kernel for `jobs_repeat` identical jobs (each on its own copy of the canvas); mirrors
    enqueue_locked / make_job (ifb_engine.cu).  in_xoff: the input window starts that many pixels into a wider bitmap (the TMA
    descriptor's base is then the 16-byte aligned address before it).  Returns the result canvases, or None if the geometry is not
    a ring-kernel geometry."""
    ih, iw = inp.shape[:2]
    w = canvas.shape[1] - x if w is None else w
    h = canvas.shape[0] - y if h is None else h
    info, blob = hv_plan(ifb, iw, ih, w, h, filter, sharpen, strip_cols, n_bands, alpha_meaningful)      # n_bands = band PAIRS
    if blob is None:
        return None
    t_lin, t_srgb, lut = transfer_tables(ifb)
    assert lib.emu_hv_sizeof_jobdev() == C.sizeof(JobDev)
    # the input as a window of a wider, 16-byte aligned bitmap
    pitch = ((iw + in_xoff) * 4 + 63) // 64 * 64
    wide = np.zeros((ih, pitch), np.uint8)
    wide[:, in_xoff * 4:(in_xoff + iw) * 4] = np.ascontiguousarray(inp).reshape(ih, iw * 4)
    assert wide.ctypes.data % 16 == 0
    outs = [np.ascontiguousarray(canvas.copy()) for _ in range(jobs_repeat)]
    jobs = (JobDev * jobs_repeat)()
    ch = 4 if alpha_meaningful else 3
    simple = compose == 0 and color_matrix is None
    for j, o in zip(jobs, outs):
        j.in_ = wide.ctypes.data + in_xoff * 4; j.out = o.ctypes.data + y * o.strides[0] + x * 4
        j.in_stride, j.out_stride, j.in_xoff = pitch, o.strides[0], in_xoff
        set_job_store(j, t_lin, t_srgb, linear=linear, alpha_meaningful=alpha_meaningful, compose=compose, matte=matte, color_matrix=color_matrix)
    in_ptrs = (C.c_void_p * jobs_repeat)(*[wide.ctypes.data] * jobs_repeat)
    in_whs = np.array([iw + in_xoff, ih, pitch] * jobs_repeat, np.uint32)
    offs = np.array([info.o_strips, info.o_hw, info.o_hdone, info.o_vw, info.o_vdone, info.o_bands, info.total], np.uint64)
    dims = np.array([iw, ih, w, h, info.cap_px], np.uint32)
    bad = lib.emu_hv_launch(info.av, ch, int(simple), grid, C.cast(jobs, C.c_void_p), jobs_repeat, C.cast(in_ptrs, C.c_void_p), in_whs.ctypes.data,
                            t_lin.ctypes.data, t_srgb.ctypes.data, lut.ctypes.data, blob.ctypes.data, offs.ctypes.data, dims.ctypes.data,
                            info.n_strips, info.n_bands, sb_low16)
    assert bad == 0, f"{bad} bad shared-memory accesses / barrier states"
    return outs
