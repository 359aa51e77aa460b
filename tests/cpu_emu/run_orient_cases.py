"""python -m tests.cpu_emu.run_orient_cases <liborient_emu.so> [n_launches]: the emulated orient_kernel
(tests/cpu_emu/orient_kernel_emu.cc, with the product's planner) against the closed form of tests/orient_oracle.py.  Also the body of
the AddressSanitizer run (the test starts it in a subprocess with libasan preloaded).

Every launch mixes jobs of all eight flags (and flags outside 2..8), in place and out of place, at sizes that straddle the 32-pixel
tile (31, 32, 33, 1 x N, N x 1, random).  Each window lies inside an exactly sized bitmap of its own (no byte after the last pixel of
the last row), full of random sentinel bytes, at a random origin and with a row pitch that is often not a multiple of 16, so that row
bases fall at every 4-byte phase modulo 16.  Per launch:
  - every bitmap equals the expected one (the result in the output window; every other byte, stride padding included, unchanged);
  - no pixel is stored twice, and the pixels stored are exactly the output window (in place: the pixels the flip moves);
  - no pixel is loaded twice, and every load is in the input window (in place: among the pixels the flip moves);
  - no shared-memory index falls outside the tile."""
import ctypes as C
import sys

import numpy as np

from imageflow_b200._lib import OrientDesc
from tests import orient_oracle as oo

SOURCES = ("orient_kernel_emu.cc", "ifb_orient.cc")          # of tests.cpu_emu.build
SIZES = [(1, 1), (1, 7), (7, 1), (5, 3), (31, 31), (32, 32), (33, 33), (31, 33), (33, 32), (1, 40), (40, 1), (65, 2), (2, 65)]


def load(so):
    L = C.CDLL(so)
    L.emu_orient.restype = C.c_long
    L.emu_orient.argtypes = [C.POINTER(OrientDesc), C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                             C.POINTER(C.c_size_t), C.POINTER(C.c_long), C.POINTER(C.c_size_t), C.c_char_p, C.c_size_t, C.c_int]
    L.emu_orient_plan.restype = C.c_long
    L.emu_orient_plan.argtypes = [C.POINTER(OrientDesc), C.c_size_t, C.POINTER(C.c_size_t)]
    return L


class Bitmap:
    """an exactly sized bitmap of sentinel bytes (its last row has no padding), 64-byte aligned, and the expected copy of it"""

    def __init__(self, rng, bw, bh, pitch):
        self.pitch = pitch
        n = (bh - 1) * pitch + bw * 4
        raw = np.empty(n + 64, np.uint8)
        off = (-raw.ctypes.data) % 64
        self.buf = raw[off:off + n]
        self.buf[:] = rng.integers(0, 256, n, dtype=np.uint8)
        self.exp = self.buf.copy()

    def view(self, arr, x, y, w, h):
        """the (h, w, 4) window of arr (buf or exp) at (x, y)"""
        return np.lib.stride_tricks.as_strided(arr[y * self.pitch + x * 4:], (h, w, 4), (self.pitch, 4, 1))

    def addrs(self, x, y, w, h, mask=None):
        yy, xx = np.indices((h, w))
        a = self.buf.ctypes.data + (y + yy) * self.pitch + (x + xx) * 4
        return set((a if mask is None else a[mask]).ravel().tolist())


def window_in(rng, w, h):
    """a bitmap holding a w x h window at a random origin, and that origin"""
    ox, oy = int(rng.integers(0, 4)), int(rng.integers(0, 3))
    bw, bh = w + ox + int(rng.integers(0, 4)), h + oy + int(rng.integers(0, 3))
    pitch = bw * 4 + 4 * int(rng.choice([0, 0, 1, 2, 3, 4, 5]))
    if rng.random() < 0.4:
        pitch = (pitch + 15) // 16 * 16
    return Bitmap(rng, bw, bh, pitch), ox, oy


def make_job(rng, o=None, in_place=None, size=None):
    """-> (desc dict, [bitmaps], {allowed loads}, {wanted stores}); the bitmaps' `exp` already holds the expected result"""
    o = int(rng.choice([1, 2, 3, 4, 5, 6, 7, 8, 0, 9, -1])) if o is None else o
    w, h = SIZES[int(rng.integers(0, len(SIZES)))] if size is None and rng.random() < 0.6 else \
        (size or (int(rng.integers(1, 70)), int(rng.integers(1, 50))))
    t = o in (5, 6, 7, 8)
    in_place = (not t and rng.random() < 0.4) if in_place is None else in_place
    src, ix, iy = window_in(rng, w, h)
    want = oo.gather(src.view(src.buf, ix, iy, w, h).copy(), o)
    d = {"in_": src.buf.ctypes.data + iy * src.pitch + ix * 4, "in_w": w, "in_h": h, "in_stride": src.pitch, "orientation": o}
    if in_place:
        d.update(out=d["in_"], out_stride=src.pitch)
        src.view(src.exp, ix, iy, w, h)[...] = want
        moved = _moved(w, h, o)
        return d, [src], src.addrs(ix, iy, w, h, moved), src.addrs(ix, iy, w, h, moved)
    ow, oh = (h, w) if t else (w, h)
    dst, dx, dy = window_in(rng, ow, oh)
    d.update(out=dst.buf.ctypes.data + dy * dst.pitch + dx * 4, out_stride=dst.pitch)
    dst.view(dst.exp, dx, dy, ow, oh)[...] = want
    return d, [src, dst], src.addrs(ix, iy, w, h), dst.addrs(dx, dy, ow, oh)


def _moved(w, h, o):
    """the pixels of a w x h window that an in-place flip o moves (not its fixed points)"""
    y, x = np.indices((h, w))
    idx = (x + w * y)[..., None].astype(np.int64)
    return oo.gather(idx, o)[..., 0] != idx[..., 0]


def descs_of(jobs):
    arr = (OrientDesc * len(jobs))()
    for desc, (d, *_rest) in zip(arr, jobs):
        for k, v in d.items():
            setattr(desc, k, v)
    return arr


def launch(L, jobs, sabotage=0):
    """runs one call of the jobs on the emulator; -> (ctas, loads, stores, bad shared-memory indices, items, error message)"""
    arr = descs_of(jobs)
    cap = sum(b.buf.size for _, bms, _, _ in jobs for b in bms) // 2 + 64
    loads, stores = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    nl, ns, bad, ni = C.c_size_t(), C.c_size_t(), C.c_long(), C.c_size_t()
    err = C.create_string_buffer(256)
    ctas = L.emu_orient(arr, len(jobs), loads.ctypes.data, stores.ctypes.data, cap, C.byref(nl), C.byref(ns), C.byref(bad), C.byref(ni),
                        err, 256, sabotage)
    assert nl.value <= cap and ns.value <= cap
    return ctas, loads[:nl.value].tolist(), stores[:ns.value].tolist(), bad.value, ni.value, err.value.decode()


def check(jobs, ctas, ld, st, bad):
    """the properties of the module docstring; raises AssertionError"""
    assert ctas >= 0 and bad == 0, (ctas, bad)
    allowed, want_st = set(), set()
    for _, _, reads, writes in jobs:
        allowed |= reads
        want_st |= writes
    assert len(set(st)) == len(st), "a pixel stored twice"
    assert set(st) == want_st, "stored set differs from the output window"
    assert len(set(ld)) == len(ld), "a pixel loaded twice"
    assert set(ld) <= allowed, "a load outside the input window"
    for _, bms, _, _ in jobs:
        for b in bms:
            diff = np.nonzero(b.buf != b.exp)[0]
            assert diff.size == 0, ("bytes differ", diff[:4].tolist())


def make_launch(rng, n=None):
    return [make_job(rng) for _ in range(int(rng.integers(1, 9)) if n is None else n)]


def run(so, n_launches=300, seed=1):
    L = load(so)
    rng = np.random.default_rng(seed)
    cases = 0
    # every flag, in place and out of place, at every listed size, then random mixed launches
    fixed = [[make_job(rng, o, ip, s) for o in range(1, 9) for ip in ((False, True) if o <= 4 else (False,))] for s in SIZES]
    for it, jobs in enumerate(fixed + [make_launch(rng) for _ in range(n_launches)]):
        ctas, ld, st, bad, _, err = launch(L, jobs)
        assert not err, err
        try:
            check(jobs, ctas, ld, st, bad)
        except AssertionError as e:
            raise AssertionError((it, [j[0] for j in jobs], e.args))
        cases += len(jobs)
    return cases


def sabotage_caught(so, kind, seed=2):
    """True when the checks above reject the launch whose plan was corrupted in way `kind` (orient_kernel_emu.cc)"""
    L = load(so)
    rng = np.random.default_rng(seed)
    jobs = [make_job(rng, o, False, (33, 31)) for o in (6, 3, 5, 2)]
    ctas, ld, st, bad, _, err = launch(L, jobs, sabotage=kind)
    try:
        check(jobs, ctas, ld, st, bad)
    except AssertionError:
        return True
    return False


if __name__ == "__main__":
    print("cases bit-exact:", run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 300))
