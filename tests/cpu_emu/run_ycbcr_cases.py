"""python -m tests.cpu_emu.run_ycbcr_cases <libycbcr_kernel_emu.so> [n_launches]: the emulated ycbcr_to_bgra_kernel
(tests/cpu_emu/ycbcr_kernel_emu.cc, with the product's planner) against tests/ycbcr_oracle.py.  Also the body of the AddressSanitizer
run (the test starts it in a subprocess with libasan preloaded).

Every launch holds several jobs.  Each plane and destination lies inside an exactly sized bitmap of its own (no byte after the last
row's window unless a random tail), full of random sentinel bytes, at a chosen byte origin and with a row pitch that is often not a
multiple of 16, so that rows start at every phase modulo 16.  The fixed launches run every sampling at every plane byte phase modulo
16, every destination 4-byte phase and widths 1..40 with heights 1..6 (chroma planes of one and two columns and rows included); items
of several CTAs whose CTA boundaries fall inside a band (a 4:2:0 row pair); random launches mix samplings and sizes.  Per launch:
  - every bitmap equals the expected one (the oracle's result in the destination window; every other byte, stride padding included,
    unchanged);
  - every destination byte is stored exactly once, and nothing else is stored;
  - every load lies in a plane of the job (the halo reads at the planes' edges included)."""
import ctypes as C
import sys

import numpy as np

from imageflow_b200._lib import YcbcrDesc
from tests import ycbcr_oracle as yo
from tests.cpu_emu.run_pixel_convert_cases import rows_in

SOURCES = ("ycbcr_kernel_emu.cc", "ifb_ycbcr.cc", "ifb_pixel_convert.cc")          # of tests.cpu_emu.build
CTA_UNITS = 2048                                                                    # ifb::kYcCtaUnits (ifb_ycbcr.h)


def load(so):
    L = C.CDLL(so)
    L.emu_ycbcr.restype = C.c_long
    L.emu_ycbcr.argtypes = [C.POINTER(YcbcrDesc), C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t),
                            C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_char_p, C.c_size_t, C.c_int]
    L.emu_ycbcr_plan.restype = C.c_long
    L.emu_ycbcr_plan.argtypes = [C.POINTER(YcbcrDesc), C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p, C.c_size_t]
    return L


def make_job(rng, sampling=None, w=None, h=None, phases=None, dphase=None):
    """-> (desc dict, [Rows], {allowed load addresses}, {wanted store addresses}); `exp` of the destination Rows holds the result.
    phases: the Y, Cb and Cr planes' first-byte phases modulo 16."""
    sampling = int(rng.choice(yo.SAMPLINGS)) if sampling is None else sampling
    w = int(rng.integers(1, 41)) if w is None else w
    h = int(rng.integers(1, 7)) if h is None else h
    phases = [int(p) for p in rng.integers(0, 16, 3)] if phases is None else phases
    dphase = 4 * int(rng.integers(0, 4)) if dphase is None else dphase
    ch, cw = yo.chroma_shape(sampling, w, h)
    py = rows_in(rng, w, h, 1, phases[0])
    pb = rows_in(rng, cw, ch, 1, phases[1])
    pr = rows_in(rng, cw, ch, 1, phases[2])
    t = rows_in(rng, w, h, 4, dphase, align4=True)
    planes = [p.view(p.buf)[..., 0].copy() for p in (py, pb, pr)]
    t.view(t.exp)[...] = yo.convert(sampling, *planes)
    d = dict(sampling=sampling, y=py.ptr, y_stride=py.pitch, cb=pb.ptr, cb_stride=pb.pitch, cr=pr.ptr, cr_stride=pr.pitch,
             dst=t.ptr, dst_stride=t.pitch, w=w, h=h)
    return d, [py, pb, pr, t], py.addrs() | pb.addrs() | pr.addrs(), t.addrs()


def descs_of(jobs):
    arr = (YcbcrDesc * len(jobs))()
    for desc, (d, *_rest) in zip(arr, jobs):
        for k, v in d.items():
            setattr(desc, k, v)
    return arr


def launch(L, jobs, sabotage=0):
    """runs one call of the jobs on the emulator; -> (ctas, [load (address << 8 | width)], [store ...], items, error)"""
    arr = descs_of(jobs)
    cap = 8 * sum(r.buf.size for _, rs, _, _ in jobs for r in rs) + 64
    loads, stores = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    nl, ns, ni = C.c_size_t(), C.c_size_t(), C.c_size_t()
    err = C.create_string_buffer(256)
    ctas = L.emu_ycbcr(arr, len(jobs), loads.ctypes.data, stores.ctypes.data, cap, C.byref(nl), C.byref(ns), C.byref(ni), err, 256,
                       sabotage)
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
    assert set((ld >> 8).tolist()) <= allowed, "a load outside the planes"
    for _, rs, _, _ in jobs:
        for r in rs:
            diff = np.nonzero(r.buf != r.exp)[0]
            assert diff.size == 0, ("bytes differ", diff[:4].tolist())


def fixed_launches(rng):
    """every sampling at every plane phase and destination phase; widths 1..40 and heights 1..6; items whose CTA boundaries fall
    inside a band; all three samplings and several sizes in one call"""
    out = []
    for s in yo.SAMPLINGS:
        jobs = [make_job(rng, s, w=1 + (i * 7) % 40, h=1 + i % 6, phases=[i % 16, (i * 5 + 3) % 16, (i * 11 + 7) % 16],
                         dphase=4 * (i % 4)) for i in range(48)]
        out += [jobs[i:i + 8] for i in range(0, len(jobs), 8)]
        out.append([make_job(rng, s, w=w, h=h) for w in (1, 2, 3, 4, 5) for h in (1, 2, 3, 4)])
    for w in range(1, 41):                                      # every width, each sampling once, mixed in one call
        out.append([make_job(rng, s, w=w, h=1 + w % 5) for s in yo.SAMPLINGS])
    # several CTAs per item: 37 or 38 groups per row (w = 147 at dphase 4..12 or 0) do not divide CTA_UNITS, so boundaries fall inside
    # a band -- at 4:2:0 between the groups of one row pair
    out.append([make_job(rng, s, w=147, h=2 * 57 + 1, dphase=4 * (s + 1)) for s in yo.SAMPLINGS])
    return out


def run(so, n_launches=200, seed=1):
    L = load(so)
    rng = np.random.default_rng(seed)
    cases = 0
    randoms = [[make_job(rng) for _ in range(int(rng.integers(1, 9)))] for _ in range(n_launches)]
    for it, jobs in enumerate(fixed_launches(rng) + randoms):
        ctas, ld, st, _, err = launch(L, jobs)
        assert not err, err
        try:
            check(jobs, ctas, ld, st)
        except AssertionError as e:
            raise AssertionError((it, [j[0] for j in jobs], e.args))
        cases += len(jobs)
    return cases


def narrow_accesses(so, sampling, w=301, h=4, phases=(5, 3, 7), dphase=8, seed=3):
    """(word or wider loads, byte loads, row count) of one job: only a row's ragged ends may take byte loads"""
    L = load(so)
    rng = np.random.default_rng(seed)
    jobs = [make_job(rng, sampling, w=w, h=h, phases=list(phases), dphase=dphase)]
    ctas, ld, st, _, err = launch(L, jobs)
    assert not err, err
    width = ld & 0xff
    return int((width >= 4).sum()), int((width == 1).sum()), h


def sabotage_caught(so, kind, seed=2):
    """True when the checks above reject the launch whose plan was corrupted in way `kind` (ycbcr_kernel_emu.cc)"""
    L = load(so)
    rng = np.random.default_rng(seed)
    jobs = [make_job(rng, s, w=33, h=5) for s in yo.SAMPLINGS]
    ctas, ld, st, _, err = launch(L, jobs, sabotage=kind)
    assert not err, err
    try:
        check(jobs, ctas, ld, st)
    except AssertionError:
        return True
    return False


if __name__ == "__main__":
    print("cases bit-exact:", run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 200))
