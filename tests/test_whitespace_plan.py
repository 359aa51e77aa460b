"""The host planner of ifb200_batch_detect_content_many (imageflow_b200/csrc/ifb_whitespace.cc) against a restatement in Python of the
reference's full-scan grid (graphics/whitespace.rs:220-281 search_rect, :333-421 check_region): origin, window sizes, window rows and
columns, and each column's range before and after the shift back inside the frame.  Also the batched entry point's validation: every
rejected descriptor with its message and status, and nothing planned or launched.  No GPU."""
import ctypes as C
import math

import numpy as np
import pytest

from imageflow_b200._lib import DetectContentDesc
from tests import cpu_emu
from tests.cpu_emu import run_whitespace_many_cases as rw


def f32(v):
    return float(np.float32(v))


def grid(w, h):
    """(y1, y2, wh, rows, [(bx, ex, xa, xb)]) of the full scan of a w x h frame (w, h >= 3), or None when it has no window"""
    at = lambda f, n: min(n, int(math.floor(f32(f32(f) * f32(n - 1)))))
    x1, x2, y1, y2 = at(0, w), at(1, w), at(0, h), at(1, h)
    if x1 == x2 or y1 == y2:
        return None
    while y2 - y1 < 7 and (y1 > 0 or y2 < h):
        y1 = max(0, y1 - 1); y2 = min(h, y2 + 1)
    while x2 - x1 < 7 and (x1 > 0 or x2 < w):
        x1 = max(0, x1 - 1); x2 = min(w, x2 + 1)
    rw_, rh = x2 - x1, y2 - y1
    ww = min(rw_, 2048 // 7)
    wh = min(rh, 2048 // ww)
    if ww <= 2 or wh <= 2:
        return None
    rows = math.ceil(f32(f32(rh) / f32(wh - 2)))
    ncols = math.ceil(f32(f32(rw_) / f32(ww - 2)))
    cols = []
    for i in range(ncols):
        bx = x1 + (ww - 2) * i
        bw = min(max(3, (x2 - bx) % 2**32), ww)
        c = (bx, bx + bw)
        if bx + bw > w:
            bx, bw = (w - bw, bw) if bw <= w else (0, w)
        cols.append(c + (bx + 1, bx + bw - 1))
    return y1, y2, wh, rows, cols


SIZES = ([(w, h) for w in range(3, 11) for h in range(3, 11)]
         + [(290 * k + 1 + r, h) for k in (1, 2, 3, 14) for r in range(4) for h in (3, 7, 20)]
         + [(w, h) for w in range(3, 41) for h in (200, 683, 1999, 2000)]
         + [(w, h) for w in (600, 1165, 3840, 7680, 20001) for h in (3, 4, 8, 11)]
         + [(h, w) for w in range(3, 41, 7) for h in (300, 1024, 2161)])


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return rw.load(cpu_emu.build(str(tmp_path_factory.mktemp("ws_plan")), *rw.SOURCES))


def test_planner_grid_matches_the_reference_arithmetic(emu):
    dummy = np.zeros(16, np.uint32)
    for w, h in SIZES:
        d = DetectContentDesc(); d.px, d.w, d.h, d.stride, d.threshold = dummy.ctypes.data, w, h, w * 4, 1
        grids = np.zeros(7, np.uint32); cols = np.zeros((4096, 4), np.uint32); nc = C.c_size_t()
        k = emu.emu_detect_content_plan(C.byref(d), 1, grids.ctypes.data, cols.ctypes.data, 4096, C.byref(nc))
        want = grid(w, h)
        assert k == 1, (w, h)
        if want is None:
            assert grids[5] == 0, (w, h)
            continue
        y1, y2, wh, rows, wc = want
        assert tuple(int(v) for v in grids) == (w, h, y1, y2, wh, rows, len(wc)), (w, h)
        assert [tuple(int(v) for v in c) for c in cols[:nc.value]] == wc, (w, h)
        # the interiors of a window row leave no gap; only the last ones may overlap those before them (all of them when w < 7)
        for i in range(1, len(wc)):
            assert wc[i - 1][2] <= wc[i][2] <= wc[i - 1][3], (w, h, i)
            assert wc[i][2] == wc[i - 1][3] or wc[i][3] == wc[-1][3], (w, h, i)


def test_frames_below_three_pixels_are_not_planned(emu):
    dummy = np.zeros(64, np.uint32)
    for w, h in [(1, 1), (2, 9), (9, 2), (1, 100), (100, 1)]:
        d = DetectContentDesc(); d.px, d.w, d.h, d.stride = dummy.ctypes.data, w, h, w * 4
        grids = np.zeros(7, np.uint32); cols = np.zeros((4, 4), np.uint32); nc = C.c_size_t()
        assert emu.emu_detect_content_plan(C.byref(d), 1, grids.ctypes.data, cols.ctypes.data, 4, C.byref(nc)) == 0


def _bad_descs(buf):
    p = buf.ctypes.data
    good = dict(px=p, w=8, h=8, stride=32, alpha_meaningful=1, threshold=1)
    return [
        (dict(good, px=0), "null bitmap pointer"),
        (dict(good, w=0), "empty bitmap"),
        (dict(good, h=0), "empty bitmap"),
        (dict(good, stride=28), "stride smaller than a BGRA row or not a multiple of 4"),
        (dict(good, stride=34), "stride smaller than a BGRA row or not a multiple of 4"),
        (dict(good, px=p + 2), "bitmap pointer not 4-byte aligned"),
        (dict(good, h=0x80000000), "oversized bitmap"),
        (dict(good, threshold=0x80000000), "threshold out of range"),
    ], good


def test_every_rejected_descriptor_is_reported_and_nothing_runs(emu):
    buf = np.zeros(64 * 64, np.uint32)
    bad, good = _bad_descs(buf)
    for fields, msg in bad:
        for pos in (0, 2):
            descs = [good, good, good]
            descs[pos] = fields
            arr = (DetectContentDesc * 3)()
            for d, f in zip(arr, descs):
                for k, v in f.items():
                    setattr(d, k, v)
            rects = np.full((3, 4), 7, np.uint32); vis = np.full(3, 7, np.uint64)
            la, b, ok, unw = C.c_int(-1), C.c_int(), C.c_int(), C.c_uint64()
            err = C.create_string_buffer(256)
            r = emu.emu_detect_content_many(arr, 3, rects.ctypes.data, vis.ctypes.data, C.byref(la), C.byref(b), C.byref(ok), C.byref(unw), err, 256)
            assert r == -1 and err.value.decode() == f"detect_content job {pos}: {msg}", (r, err.value, msg)
            assert la.value == -1 and (rects == 7).all() and (vis == 7).all()         # nothing launched, nothing written
