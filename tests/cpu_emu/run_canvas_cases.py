"""python -m tests.cpu_emu.run_canvas_cases <libcanvas_emu.so> [n_launches]: the emulated canvas_kernel
(tests/cpu_emu/canvas_kernel_emu.cc, with the product's planner) against the numpy oracle (tests/canvas_oracle.py).  Also the body
of the AddressSanitizer run (the test starts it in a subprocess with libasan preloaded).

Every launch mixes jobs of all four ops.  Each job's windows lie inside bitmaps of their own, exactly sized (no byte after the last
pixel of the last row), full of random sentinel bytes, at random origins and with row pitches that are not always multiples of 16,
so that rows start at every phase modulo 16 bytes and a copy's source and destination often differ in phase.  Per launch:
  - every bitmap equals the oracle's (results, and every byte outside the windows and in the stride padding unchanged);
  - no pixel is stored twice;
  - the pixels stored are exactly the pixels the oracle writes;
  - the pixels loaded are copy sources or pixels normalised in place, each loaded at most once."""
import ctypes as C
import sys

import numpy as np

from imageflow_b200._lib import CanvasDesc
from tests import canvas_oracle as co

SOURCES = ("canvas_kernel_emu.cc", "ifb_canvas.cc")          # of tests.cpu_emu.build
FILL, COPY, EXPAND, NORMALIZE = range(4)


def load(so):
    L = C.CDLL(so)
    L.emu_canvas.restype = C.c_long
    L.emu_canvas.argtypes = [C.POINTER(CanvasDesc), C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                             C.POINTER(C.c_size_t), C.c_char_p, C.c_size_t, C.c_int]
    return L


class Bitmap:
    """an exactly sized bitmap of sentinel bytes (its last row has no padding) and the oracle's copy of it"""

    def __init__(self, rng, bw, bh, pitch):
        self.pitch = pitch
        self.buf = rng.integers(0, 256, (bh - 1) * pitch + bw * 4, dtype=np.uint8)
        self.buf[3::4][rng.random(self.buf[3::4].size) < 0.3] = 255
        self.exp = self.buf.copy()
        self.mask = np.zeros(self.buf.size // 4, bool)

    def win(self, x, y, w, h, am, expected=True):
        return co.Win(self.exp if expected else self.buf, y * self.pitch + x * 4, w, h, self.pitch, am, self.mask if expected else None)

    def addr(self, word_mask):
        return set((self.buf.ctypes.data + 4 * np.nonzero(word_mask)[0]).tolist())

    def region_mask(self, win):
        m = np.zeros_like(self.mask)
        win.mark(mask=m)
        return m


def window_in(rng, w, h):
    """a bitmap holding a w x h window at a random origin, and that origin"""
    ox, oy = int(rng.integers(0, 4)), int(rng.integers(0, 3))
    bw, bh = w + ox + int(rng.integers(0, 4)), h + oy + int(rng.integers(0, 3))
    pitch = bw * 4 + 4 * int(rng.choice([0, 0, 1, 2, 3, 4, 5]))
    if rng.random() < 0.4:
        pitch = (pitch + 15) // 16 * 16
    return Bitmap(rng, bw, bh, pitch), ox, oy


def color(rng):
    c = [int(v) for v in rng.integers(0, 256, 4)]
    r = rng.random()
    if r < 0.4:
        c[3] = 255
    elif r < 0.5:
        c = [0, 0, 0, 0]
    elif r < 0.6:
        c[3] = 0                                      # alpha 0 with colour bytes: filled as they are
    return c


def make_job(rng, big=False):
    """-> (fill a CanvasDesc, apply the oracle, [bitmaps], {allowed load addresses})"""
    op = int(rng.integers(0, 4))
    lim = 90 if big else 23
    w, h = int(rng.integers(1, lim)), int(rng.integers(1, lim // 2 + 2))
    am, in_am = bool(rng.random() < 0.5), bool(rng.random() < 0.5)
    cv, ox, oy = window_in(rng, w, h)
    d = {"op": op, "px": cv.buf.ctypes.data + oy * cv.pitch + ox * 4, "w": w, "h": h, "stride": cv.pitch, "alpha_meaningful": int(am)}
    bms, reads = [cv], set()
    if op == FILL:
        if rng.random() < 0.1:                        # zero size, anywhere: a no-op
            x1, y1 = int(rng.integers(0, 3 * w)), int(rng.integers(0, 3 * h))
            x2, y2 = (x1, int(rng.integers(0, 3 * h))) if rng.random() < 0.5 else (int(rng.integers(0, 3 * w)), y1)
        else:
            x1, x2 = sorted(int(v) for v in rng.choice(w + 1, 2, replace=False))
            y1, y2 = sorted(int(v) for v in rng.choice(h + 1, 2, replace=False))
        c = color(rng)
        d.update(x1=x1, y1=y1, x2=x2, y2=y2, color_bgra=c)
        oracle = lambda: co.fill_rectangle(cv.win(ox, oy, w, h, am), c, x1, y1, x2, y2)
    elif op == NORMALIZE:
        oracle = lambda: co.normalize_unused_alpha(cv.win(ox, oy, w, h, am))
        if not am:
            reads |= cv.addr(cv.region_mask(cv.win(ox, oy, w, h, am)))
    elif op == COPY:
        iw, ih = int(rng.integers(1, lim)), int(rng.integers(1, lim // 2 + 2))
        src, ix, iy = window_in(rng, iw, ih)
        cw, ch = int(rng.integers(1, min(w, iw) + 1)), int(rng.integers(1, min(h, ih) + 1))
        fx, fy = int(rng.integers(0, iw - cw + 1)), int(rng.integers(0, ih - ch + 1))
        tx, ty = int(rng.integers(0, w - cw + 1)), int(rng.integers(0, h - ch + 1))
        d.update(in_=src.buf.ctypes.data + iy * src.pitch + ix * 4, in_w=iw, in_h=ih, in_stride=src.pitch, in_alpha_meaningful=int(in_am),
                 x1=fx, y1=fy, x2=tx, y2=ty, cw=cw, ch=ch)
        bms.append(src)
        oracle = lambda: co.copy_rectangle(src.win(ix, iy, iw, ih, in_am), cv.win(ox, oy, w, h, am), fx, fy, tx, ty, cw, ch)
        reads |= src.addr(src.region_mask(src.win(ix + fx, iy + fy, cw, ch, in_am)))
        if in_am and not am:
            reads |= cv.addr(cv.region_mask(cv.win(ox, oy, w, h, am)))
        if am and not in_am:
            reads |= src.addr(src.region_mask(src.win(ix, iy, iw, ih, in_am)))
    else:
        iw, ih = max(1, w - int(rng.integers(0, w))), max(1, h - int(rng.integers(0, h)))
        l, t = int(rng.integers(0, w - iw + 1)), int(rng.integers(0, h - ih + 1))
        r, b = w - iw - l, h - ih - t
        src, ix, iy = window_in(rng, iw, ih)
        c = color(rng)
        d.update(in_=src.buf.ctypes.data + iy * src.pitch + ix * 4, in_w=iw, in_h=ih, in_stride=src.pitch, in_alpha_meaningful=int(in_am),
                 x1=l, y1=t, x2=r, y2=b, color_bgra=c)
        bms.append(src)
        oracle = lambda: co.expand_canvas(src.win(ix, iy, iw, ih, in_am), cv.win(ox, oy, w, h, am), l, t, r, b, c)
        reads |= src.addr(src.region_mask(src.win(ix, iy, iw, ih, in_am)))
    return d, oracle, bms, reads


def fill(desc, d):
    for k, v in d.items():
        setattr(desc, k, (C.c_uint8 * 4)(*v) if k == "color_bgra" else v)


def launch(L, jobs, sabotage=0):
    """runs one call of the jobs on the emulator; -> (ctas, loads, stores, error message)"""
    descs = (CanvasDesc * len(jobs))()
    for desc, (d, *_rest) in zip(descs, jobs):
        fill(desc, d)
    cap = sum(b.buf.size for _, _, bms, _ in jobs for b in bms) // 2 + 64
    loads, stores = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    nl, ns = C.c_size_t(), C.c_size_t()
    err = C.create_string_buffer(256)
    ctas = L.emu_canvas(descs, len(jobs), loads.ctypes.data, stores.ctypes.data, cap, C.byref(nl), C.byref(ns), err, 256, sabotage)
    assert nl.value <= cap and ns.value <= cap
    return ctas, loads[:nl.value].tolist(), stores[:ns.value].tolist(), err.value.decode()


def check(jobs, ctas, ld, st):
    """the four properties of the module docstring; raises AssertionError"""
    assert ctas >= 0
    want_st, allowed = set(), set()
    for _, _, bms, reads in jobs:
        allowed |= reads
        for b in bms:
            want_st |= b.addr(b.mask)
    assert len(set(st)) == len(st), "a pixel stored twice"
    assert set(st) == want_st, "stored set differs from the oracle's write mask"
    assert len(set(ld)) == len(ld) and set(ld) <= allowed, "a load outside the copy sources and normalised pixels"
    for _, _, bms, _ in jobs:
        for b in bms:
            bad = np.nonzero(b.buf != b.exp)[0]
            assert bad.size == 0, ("bytes differ", bad[:4].tolist())


def make_launch(rng, it):
    jobs = [make_job(rng, big=(it % 17 == 0)) for _ in range(int(rng.integers(1, 9)))]
    for _, oracle, _, _ in jobs:
        oracle()
    return jobs


def run(so, n_launches=400, seed=1):
    L = load(so)
    rng = np.random.default_rng(seed)
    cases = 0
    for it in range(n_launches):
        jobs = make_launch(rng, it)
        ctas, ld, st, err = launch(L, jobs)
        assert not err, err
        try:
            check(jobs, ctas, ld, st)
        except AssertionError as e:
            raise AssertionError((it, [j[0] for j in jobs], e.args))
        cases += len(jobs)
    return cases


def sabotage_caught(so, kind, seed=2):
    """True when the checks above reject the launch whose plan was corrupted in way `kind` (canvas_kernel_emu.cc)"""
    L = load(so)
    rng = np.random.default_rng(seed)
    while True:
        jobs = make_launch(rng, 1)
        if any(b.mask.any() for _, _, bms, _ in jobs for b in bms):
            break
    ctas, ld, st, err = launch(L, jobs, sabotage=kind)
    try:
        check(jobs, ctas, ld, st)
    except AssertionError:
        return True
    return False


if __name__ == "__main__":
    print("cases bit-exact:", run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 400))
