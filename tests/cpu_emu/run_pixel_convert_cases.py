"""python -m tests.cpu_emu.run_pixel_convert_cases <libpixel_convert_kernel_emu.so> [n_launches]: the emulated pixel_convert_kernel
(tests/cpu_emu/pixel_convert_kernel_emu.cc, with the product's planner) against tests/pixel_convert_oracle.py.  Also the body of the
AddressSanitizer run (the test starts it in a subprocess with libasan preloaded).

Every launch holds several jobs.  Each window lies inside an exactly sized bitmap of its own (no byte after the last row's window
unless a random tail), full of random sentinel bytes, at a chosen byte origin and with a row pitch that is often not a multiple of 16,
so that rows start at every phase modulo 16.  The fixed launches run every op at every source byte phase modulo 16, every destination
4-byte phase (every byte phase for RGB24 rows) and widths 1..40; random launches mix ops, sizes, in-place swaps and opaque.  Per
launch:
  - every bitmap equals the expected one (the oracle's result in the destination window; every other byte, stride padding included,
    unchanged);
  - every destination byte is stored exactly once, and nothing else is stored;
  - every load lies in a source window (in place: in the window itself)."""
import ctypes as C
import sys

import numpy as np

from imageflow_b200._lib import PixelConvertDesc
from tests import pixel_convert_oracle as po

SOURCES = ("pixel_convert_kernel_emu.cc", "ifb_pixel_convert.cc")          # of tests.cpu_emu.build


def load(so):
    L = C.CDLL(so)
    L.emu_pixel_convert.restype = C.c_long
    L.emu_pixel_convert.argtypes = [C.POINTER(PixelConvertDesc), C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                                    C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_char_p, C.c_size_t, C.c_int]
    L.emu_pixel_convert_plan.restype = C.c_long
    L.emu_pixel_convert_plan.argtypes = [C.POINTER(PixelConvertDesc), C.c_size_t, C.POINTER(C.c_size_t)]
    return L


class Rows:
    """a w x h window of `ch`-byte pixels at byte `off` of an exactly sized, 64-byte aligned buffer of sentinel bytes, with its
    expected copy"""

    def __init__(self, rng, w, h, ch, off, pitch, tail=0):
        self.w, self.h, self.ch, self.off, self.pitch = w, h, ch, off, pitch
        n = off + (h - 1) * pitch + w * ch + tail
        raw = np.empty(n + 64, np.uint8)
        a = (-raw.ctypes.data) % 64
        self.buf = raw[a:a + n]
        self.buf[:] = rng.integers(0, 256, n, dtype=np.uint8)
        self.exp = self.buf.copy()

    @property
    def ptr(self):
        return self.buf.ctypes.data + self.off

    def view(self, arr):
        return np.lib.stride_tricks.as_strided(arr[self.off:], (self.h, self.w, self.ch), (self.pitch, self.ch, 1))

    def addrs(self):
        y, x = np.indices((self.h, self.w * self.ch))
        return set((self.ptr + y * self.pitch + x).ravel().tolist())


def rows_in(rng, w, h, ch, phase, align4=False):
    """Rows whose first byte lies at `phase` modulo 16, with a random pitch (a multiple of 4 when align4)"""
    pad = int(rng.choice([0, 0, 1, 2, 3, 5, 7, 13]))
    pitch = w * ch + (pad * 4 if align4 else pad)
    if rng.random() < 0.3:
        pitch = (pitch + 15) // 16 * 16
    return Rows(rng, w, h, ch, phase + 16 * int(rng.integers(0, 3)), pitch, int(rng.integers(0, 4)))


def make_job(rng, op=None, w=None, h=None, sphase=None, dphase=None, in_place=None, opaque=None):
    """-> (desc dict, [Rows], {allowed load addresses}, {wanted store addresses}); `exp` of the Rows already holds the result"""
    op = int(rng.choice(po.OPS)) if op is None else op
    cs, cd = po.CHANNELS[op]
    w = int(rng.integers(1, 41)) if w is None else w
    h = int(rng.integers(1, 6)) if h is None else h
    opaque = bool(rng.random() < 0.5) if opaque is None else opaque
    in_place = (op == po.RGBA_TO_BGRA and rng.random() < 0.3) if in_place is None else in_place
    if dphase is None:
        dphase = 4 * int(rng.integers(0, 4)) if cd == 4 else int(rng.integers(0, 16))
    if in_place:
        r = rows_in(rng, w, h, 4, dphase, align4=True)
        want = po.convert(op, r.view(r.buf).copy(), opaque)
        r.view(r.exp)[...] = want
        d = dict(op=op, src=r.ptr, src_stride=r.pitch, dst=r.ptr, dst_stride=r.pitch, w=w, h=h, opaque=int(opaque))
        return d, [r], r.addrs(), r.addrs()
    sphase = int(rng.integers(0, 16)) if sphase is None else sphase
    s = rows_in(rng, w, h, cs, sphase)
    t = rows_in(rng, w, h, cd, dphase, align4=cd == 4)
    t.view(t.exp)[...] = po.convert(op, s.view(s.buf).copy(), opaque)
    d = dict(op=op, src=s.ptr, src_stride=s.pitch, dst=t.ptr, dst_stride=t.pitch, w=w, h=h, opaque=int(opaque))
    return d, [s, t], s.addrs(), t.addrs()


def descs_of(jobs):
    arr = (PixelConvertDesc * len(jobs))()
    for desc, (d, *_rest) in zip(arr, jobs):
        for k, v in d.items():
            setattr(desc, k, v)
    return arr


def launch(L, jobs, sabotage=0):
    """runs one call of the jobs on the emulator; -> (ctas, [(load address, width)], [(store address, width)], items, error)"""
    arr = descs_of(jobs)
    cap = 2 * sum(r.buf.size for _, rs, _, _ in jobs for r in rs) + 64
    loads, stores = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    nl, ns, ni = C.c_size_t(), C.c_size_t(), C.c_size_t()
    err = C.create_string_buffer(256)
    ctas = L.emu_pixel_convert(arr, len(jobs), loads.ctypes.data, stores.ctypes.data, cap, C.byref(nl), C.byref(ns), C.byref(ni),
                               err, 256, sabotage)
    assert nl.value <= cap and ns.value <= cap
    return ctas, loads[:nl.value], stores[:ns.value], ni.value, err.value.decode()


def check(jobs, ctas, ld, st):
    """the properties of the module docstring; raises AssertionError"""
    assert ctas >= 0, ctas
    allowed, want_st = set(), set()
    for _, _, reads, writes in jobs:
        allowed |= reads
        want_st |= writes
    st_addr = (st >> 8).tolist()
    assert len(set(st_addr)) == len(st_addr), "a destination byte stored twice"
    assert set(st_addr) == want_st, "stored bytes differ from the destination windows"
    assert set((ld >> 8).tolist()) <= allowed, "a load outside the source windows"
    for _, rs, _, _ in jobs:
        for r in rs:
            diff = np.nonzero(r.buf != r.exp)[0]
            assert diff.size == 0, ("bytes differ", diff[:4].tolist())


def fixed_launches(rng):
    """every op at every source phase modulo 16 and destination phase, widths 1..40 over the jobs, 8 jobs per launch"""
    out = []
    for op in po.OPS:
        cd = po.CHANNELS[op][1]
        dphases = range(0, 16, 4) if cd == 4 else range(16)
        jobs = [make_job(rng, op, w=1 + (i * 7) % 40, h=1 + i % 3, sphase=i % 16, dphase=dphases[i % len(dphases)], in_place=False)
                for i in range(48)]
        out += [jobs[i:i + 8] for i in range(0, len(jobs), 8)]
        if op == po.RGBA_TO_BGRA:                               # in place at every 4-byte phase, opaque and not
            out.append([make_job(rng, op, w=w, sphase=0, dphase=p, in_place=True, opaque=o)
                        for w in (1, 3, 4, 5, 8, 13) for p in (0, 4, 8, 12) for o in (False, True)][:16])
    for w in range(1, 41):                                      # every width, each op once
        out.append([make_job(rng, op, w=w, h=2) for op in po.OPS])
    return out


def run(so, n_launches=200, seed=1):
    L = load(so)
    rng = np.random.default_rng(seed)
    cases = 0
    randoms = [[make_job(rng) for _ in range(int(rng.integers(1, 9)))] for _ in range(n_launches)]
    # wide rows: groups that straddle rows and CTAs of several thousand groups
    randoms.append([make_job(rng, op, w=int(rng.integers(600, 1400)), h=int(rng.integers(8, 20))) for op in po.OPS])
    for it, jobs in enumerate(fixed_launches(rng) + randoms):
        ctas, ld, st, _, err = launch(L, jobs)
        assert not err, err
        try:
            check(jobs, ctas, ld, st)
        except AssertionError as e:
            raise AssertionError((it, [j[0] for j in jobs], e.args))
        cases += len(jobs)
    return cases


def narrow_accesses(so, op, w=37, h=4, sphase=5, dphase=8, seed=3):
    """(word or wider loads, byte loads, row count) of one job: only a row's ragged ends may take byte loads"""
    L = load(so)
    rng = np.random.default_rng(seed)
    jobs = [make_job(rng, op, w=w, h=h, sphase=sphase, dphase=dphase, in_place=False, opaque=False)]
    ctas, ld, st, _, err = launch(L, jobs)
    assert not err, err
    width = ld & 0xff
    return int((width >= 4).sum()), int((width == 1).sum()), h


def sabotage_caught(so, kind, seed=2):
    """True when the checks above reject the launch whose plan was corrupted in way `kind` (pixel_convert_kernel_emu.cc)"""
    L = load(so)
    rng = np.random.default_rng(seed)
    jobs = [make_job(rng, op, w=33, h=5, in_place=False) for op in (po.RGB24_TO_BGRA, po.BGRA_TO_RGB24, po.GRAY_TO_BGRA)]
    ctas, ld, st, _, err = launch(L, jobs, sabotage=kind)
    assert not err, err
    try:
        check(jobs, ctas, ld, st)
    except AssertionError:
        return True
    return False


if __name__ == "__main__":
    print("cases bit-exact:", run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 200))
