"""python -m tests.cpu_emu.run_watermark_cases <libwatermark_emu.so> [n_calls]: the emulated watermark kernels
(tests/cpu_emu/watermark_kernel_emu.cc: vpass_f_kernel and watermark_composite_kernel with the product's planner) against the CPU
oracle.  Also the body of the AddressSanitizer run (the test starts it in a subprocess with libasan preloaded).

Every call holds several jobs.  Watermarks are sub-windows of exactly sized bitmaps of random sentinel bytes (no byte after the last
pixel of the last row) at a random origin, with row pitches that are often not multiples of 16; several jobs share a watermark, so that
groups hold several frames; opacities include none, NaN, > 1, 0 and negative ones; compose modes, formats, working spaces, filters and
zero-area jobs are mixed.  Each frame is such a bitmap too, with the draw's rectangle at a random place in it.  The H pass is the
oracle's (oracle.resample_stages), which the GPU's H pass equals bit for bit (tests/test_gpu_parity.py).  Per call:
  - every group's F, as vpass_f_kernel stores it, equals the oracle's V pass bit for bit;
  - every frame equals the node-by-node expansion (oracle.scale_and_render of the watermark after its Alpha chain, under the Compose
    rule) in the rectangle, and every other byte, stride padding included, is unchanged;
  - no pixel is stored twice, and the pixels stored are exactly the rectangles of the jobs with pixels;
  - every load of a CTA is in its own job's rectangle or in its own group's F."""
import ctypes as C
import sys

import numpy as np

import imageflow_b200 as ifb
import oracle
from imageflow_b200._lib import WatermarkDesc
from tests import color_oracle as co
from tests import watermark_oracle as wo
from tests.cpu_emu import csr, transfer_tables
from tests.cpu_emu.run_orient_cases import Bitmap, window_in

SOURCES = ("watermark_kernel_emu.cc", "ifb_watermark.cc", "ifb_orient.cc")          # of tests.cpu_emu.build
FILTERS = [2, 4, 13, 14, 6, 22]
OPACITIES = [1.0, 1.0, float("nan"), 2.5, 0.7, 0.3, 0.0, -1.0]


def load(so):
    L = C.CDLL(so)
    L.emu_watermark_plan.restype = C.c_long
    L.emu_watermark_plan.argtypes = [C.POINTER(WatermarkDesc), C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                     C.c_size_t, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_char_p, C.c_size_t]
    L.emu_watermark.restype = C.c_long
    L.emu_watermark.argtypes = [C.POINTER(WatermarkDesc), C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_char_p,
                                C.c_size_t, C.c_int]
    return L


_T = {}


def tables():
    if not _T:
        _T.update(zip(("lin", "srgb", "lut"), transfer_tables(ifb)))
    return _T


def make_watermark(rng, w=None, h=None):
    """a watermark window in a sentinel bitmap -> dict"""
    w = int(rng.integers(1, 40)) if w is None else w
    h = int(rng.integers(1, 30)) if h is None else h
    bm, x, y = window_in(rng, w, h)
    if rng.random() < 0.5:                                   # transparent content
        bm.buf[:] = np.where(rng.random(bm.buf.size) < 0.3, 0, bm.buf).astype(np.uint8)
    bm.exp[:] = bm.buf
    return {"bm": bm, "x": x, "y": y, "w": w, "h": h, "am": bool(rng.random() < 0.6)}


def make_job(rng, wm, draw=None, frame_shape=None):
    """one job drawing `wm`: draw = (w, h, filter, linear, opacity) (shared by the jobs of a group), the frame a fresh sentinel bitmap"""
    w, h, filt, linear, op = draw
    fw, fh = (w + int(rng.integers(0, 9)), h + int(rng.integers(0, 6))) if frame_shape is None else frame_shape[:2]
    bm, fx, fy = window_in(rng, fw, fh) if frame_shape is None else (frame_shape[2], 0, 0)
    x, y = int(rng.integers(0, fw - w + 1)), int(rng.integers(0, fh - h + 1))
    return {"wm": wm, "frame": bm, "fx": fx, "fy": fy, "fw": fw, "fh": fh, "x": x, "y": y, "w": w, "h": h, "filter": filt, "linear": linear,
            "opacity": op, "compose": int(rng.integers(0, 3)), "matte": tuple(int(v) for v in rng.integers(0, 256, 4))}


def random_draw(rng):
    if rng.random() < 0.05:
        return (0, int(rng.integers(1, 5)), 2, 1, 1.0)                # zero area: skipped
    return (int(rng.integers(1, 45)), int(rng.integers(1, 25)), int(rng.choice(FILTERS)), int(rng.random() < 0.7),
            float(rng.choice(OPACITIES)))


def desc_of(j):
    d = WatermarkDesc()
    wm, fb = j["wm"], j["frame"]
    d.draw.in_ = wm["bm"].buf.ctypes.data + wm["y"] * wm["bm"].pitch + wm["x"] * 4
    d.draw.in_w, d.draw.in_h, d.draw.in_stride = wm["w"], wm["h"], wm["bm"].pitch
    d.draw.canvas = fb.buf.ctypes.data + j["fy"] * fb.pitch + j["fx"] * 4
    d.draw.cv_w, d.draw.cv_h, d.draw.cv_stride = j["fw"], j["fh"], fb.pitch
    d.draw.x, d.draw.y, d.draw.w, d.draw.h = j["x"], j["y"], j["w"], j["h"]
    d.draw.filter, d.draw.linear, d.draw.alpha_meaningful, d.draw.compose = j["filter"], j["linear"], int(wm["am"]), j["compose"]
    d.draw.matte_bgra = (C.c_uint8 * 4)(*j["matte"])
    d.opacity = j["opacity"]
    return d


def source_of(wm, opacity):
    """the watermark's pixels after the node's Alpha step (watermark.rs:166-172) -> (pixels, alpha_meaningful)"""
    src = np.ascontiguousarray(wm["bm"].view(wm["bm"].buf, wm["x"], wm["y"], wm["w"], wm["h"])).copy()
    op = np.float32(opacity)
    op = op if op != op else np.float32(min(max(op, np.float32(0)), np.float32(1)))
    if not op < 1:
        return src, wm["am"]
    out, am, _ = co.run_chain(src, co.preset(co.ALPHA, float(op)), wm["am"])
    return out, am


def expect(jobs):
    for j in jobs:
        if j["w"] == 0 or j["h"] == 0:
            continue
        src, am = source_of(j["wm"], j["opacity"])
        fb = j["frame"]
        cv = fb.view(fb.exp, j["fx"], j["fy"], j["fw"], j["fh"])
        oracle.scale_and_render(src, cv, x=j["x"], y=j["y"], w=j["w"], h=j["h"], filter=j["filter"], linear=bool(j["linear"]),
                                alpha_meaningful=am, compose=wo.drawn_compose(j["compose"]), matte=j["matte"])


def plan(L, arr, n):
    t = tables()
    g, rep, opac = np.zeros(8 * n + 8, np.uint32), np.zeros(n + 1, np.uint32), np.zeros(n + 1, np.float32)
    jb = np.zeros(4 * n + 4, np.uint32)
    ng, nj = C.c_size_t(), C.c_size_t()
    err = C.create_string_buffer(256)
    ctas = L.emu_watermark_plan(arr, n, t["lin"].ctypes.data, t["srgb"].ctypes.data, g.ctypes.data, rep.ctypes.data, opac.ctypes.data,
                                n + 1, jb.ctypes.data, n + 1, C.byref(ng), C.byref(nj), err, 256)
    return ctas, g[:8 * ng.value].reshape(-1, 8), rep[:ng.value], opac[:ng.value], jb[:4 * nj.value].reshape(-1, 4), err.value.decode()


def launch(L, jobs, sabotage=0):
    """runs one call on the emulator -> (ctas, groups, loads (addr, cta), stores (addr, cta), F buffer, expected F per group, err)"""
    arr = (WatermarkDesc * max(len(jobs), 1))(*[desc_of(j) for j in jobs])
    ctas, groups, rep, _, _, err = plan(L, arr, len(jobs))
    if ctas < 0:
        return ctas, None, None, None, None, None, err
    t = tables()
    keep, inter_p, in_h, axis_p, want_f = [], [], [], [], []
    for g, r in zip(groups, rep):
        j = jobs[int(r)]
        src, am = source_of(j["wm"], j["opacity"])
        v, f = oracle.resample_stages(src, np.zeros((j["h"], j["w"], 4), np.uint8), filter=j["filter"], linear=bool(j["linear"]),
                                      alpha_meaningful=am)
        v = np.ascontiguousarray(v)
        l, rr, o, w = csr(ifb.populate_weights(j["filter"], j["h"], src.shape[0]))
        keep += [v, l, rr, o, w]
        inter_p.append(v.ctypes.data); in_h.append(src.shape[0]); axis_p += [l.ctypes.data, rr.ctypes.data, o.ctypes.data, w.ctypes.data]
        want_f.append(f)
    f_words = int(sum(int(g[0]) * int(g[1]) * 4 for g in groups)) + 4
    F = np.full(f_words, np.nan, np.float32)
    cap = 4 * sum(j["w"] * j["h"] for j in jobs) + 64
    loads, stores = np.zeros(2 * cap, np.uint64), np.zeros(2 * cap, np.uint64)
    nl, ns = C.c_size_t(), C.c_size_t()
    ebuf = C.create_string_buffer(256)
    P = lambda xs, t_: (t_ * max(len(xs), 1))(*xs)
    got = L.emu_watermark(arr, len(jobs), P(inter_p, C.c_void_p), np.array(in_h + [0], np.uint32).ctypes.data, P(axis_p, C.c_void_p),
                          F.ctypes.data, t["lin"].ctypes.data, t["srgb"].ctypes.data, t["lut"].ctypes.data, loads.ctypes.data,
                          stores.ctypes.data, cap, C.byref(nl), C.byref(ns), ebuf, 256, sabotage)
    assert got == ctas and nl.value <= cap and ns.value <= cap
    return ctas, groups, loads[:2 * nl.value].reshape(-1, 2), stores[:2 * ns.value].reshape(-1, 2), F, want_f, ""


def check(jobs, ctas, groups, ld, st, F, want_f):
    """the properties of the module docstring; raises AssertionError"""
    assert ctas >= 0
    for g, wf in zip(groups, want_f):
        w, h, off = int(g[0]), int(g[1]), int(g[7]) // 4
        assert np.array_equal(F[off:off + w * h * 4].view(np.uint32), wf.reshape(-1).view(np.uint32)), "F differs from the oracle's V pass"
    live = [j for j in jobs if j["w"] and j["h"]]
    rect = {}                                               # rectangle origin address -> (stride, w, h)
    want_st = set()
    for j in live:
        fb = j["frame"]
        o = fb.buf.ctypes.data + (j["fy"] + j["y"]) * fb.pitch + (j["fx"] + j["x"]) * 4
        rect[o] = (fb.pitch, j["w"], j["h"])
        want_st |= fb.addrs(j["fx"] + j["x"], j["fy"] + j["y"], j["w"], j["h"])
    sa = st[:, 0].tolist()
    assert len(set(sa)) == len(sa), "a pixel stored twice"
    assert set(sa) == want_st, "stored set differs from the rectangles"
    # each CTA's job and group, from the plan: CTAs run group by group, tile by tile, job by job
    firsts = groups[:, 6].astype(np.int64)
    fbase = F.ctypes.data
    outs = {}                                               # planner job index -> rectangle origin, by matching the descriptors' rects
    _, _, _, _, jb, _ = plan_cache[id(jobs)]
    for k, row in enumerate(jb):
        outs[k] = int(row[0]) | (int(row[1]) << 32)
    for addr, cta in ld.tolist():
        gi = int(np.searchsorted(firsts, cta, side="right")) - 1
        g = groups[gi]
        c = cta - int(g[6])
        job = int(g[4]) + c % int(g[5])
        f0 = fbase + int(g[7])
        if f0 <= addr < f0 + int(g[0]) * int(g[1]) * 16:
            assert (addr - f0) % 16 == 0
            continue
        o = outs[job]
        stride, w, h = rect[o]
        d = addr - o
        assert d >= 0 and d % 4 == 0 and d // stride < h and (d % stride) // 4 < w, "a load outside the job's rectangle and the group's F"
    for j in jobs:
        for bm in (j["frame"], j["wm"]["bm"]):
            diff = np.nonzero(bm.buf != bm.exp)[0]
            assert diff.size == 0, ("bytes differ", diff[:4].tolist())


plan_cache = {}


def run_call(L, jobs, sabotage=0):
    arr = (WatermarkDesc * max(len(jobs), 1))(*[desc_of(j) for j in jobs])
    plan_cache[id(jobs)] = plan(L, arr, len(jobs))
    expect(jobs)
    ctas, groups, ld, st, F, want_f, err = launch(L, jobs, sabotage)
    assert not err, err
    try:
        check(jobs, ctas, groups, ld, st, F, want_f)
    finally:
        plan_cache.pop(id(jobs), None)


def random_call(rng):
    jobs = []
    for _ in range(int(rng.integers(1, 4))):
        wm = make_watermark(rng)
        for _ in range(int(rng.integers(1, 3))):
            draw = random_draw(rng)
            jobs += [make_job(rng, wm, draw) for _ in range(int(rng.integers(1, 4)))]
    return [jobs[i] for i in rng.permutation(len(jobs))]


def run(so, n_calls=60, seed=1):
    L = load(so)
    rng = np.random.default_rng(seed)
    cases = 0
    for it in range(n_calls):
        jobs = random_call(rng)
        try:
            run_call(L, jobs)
        except AssertionError as e:
            raise AssertionError((it, e.args))
        cases += len(jobs)
    return cases


def sabotage_caught(so, kind, seed=2):
    """True when the checks above reject the call whose plan was corrupted in way `kind` (watermark_kernel_emu.cc)"""
    L = load(so)
    rng = np.random.default_rng(seed)
    a, b = make_watermark(rng, 30, 20), make_watermark(rng, 17, 9)
    a["am"] = b["am"] = True
    da, db = (24, 14, 2, 1, 0.6), (9, 11, 4, 1, 1.0)
    frames = [Bitmap(rng, 40, 30, 40 * 4 + 12) for _ in range(3)]    # one pitch for the group's frames: a moved job stays inside
    jobs = [make_job(rng, a, da, (40, 30, f)) for f in frames] + [make_job(rng, b, db)]
    for j in jobs[:3]:
        j["x"], j["y"] = 5, 6
    try:
        run_call(L, jobs, sabotage=kind)
    except AssertionError:
        return True
    return False


if __name__ == "__main__":
    print("cases bit-exact:", run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 60))
