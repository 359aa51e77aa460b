"""python -m tests.cpu_emu.run_ycbcr_enc_cases <libycbcr_enc_kernel_emu.so> [n_launches]: the emulated bgra_to_ycbcr_kernel
(tests/cpu_emu/ycbcr_enc_kernel_emu.cc, with the product's planner) against tests/ycbcr_enc_oracle.py.  Also the body of the
AddressSanitizer run (the test starts it in a subprocess with libasan preloaded).

Every launch holds several jobs.  The source and each plane lie inside an exactly sized bitmap of its own (no byte after the last
row's window unless a random tail), full of random sentinel bytes, at a chosen byte origin and with a row pitch that is often not a
multiple of 16, so that rows start at every phase modulo 16 (every 4-byte phase for the source).  The fixed launches run every sampling
at every source and plane phase, widths 1..40 with heights 1..6, items of several CTAs whose CTA boundaries fall inside a band (a 4:2:0
row pair), and matte jobs whose alpha holds 0, 255 and values between; random launches mix samplings, sizes and mattes.  Per launch:
  - every bitmap equals the expected one (the oracle's planes in the plane windows; every other byte, the source and stride padding
    included, unchanged);
  - every plane byte is stored exactly once, and nothing else is stored;
  - every load lies in the source window of a job."""
import ctypes as C
import sys

import numpy as np

from imageflow_b200._lib import BgraToYcbcrDesc
from tests import ycbcr_enc_oracle as eo
from tests.cpu_emu.run_pixel_convert_cases import Rows, rows_in

SOURCES = ("ycbcr_enc_kernel_emu.cc", "ifb_ycbcr_enc.cc", "ifb_ycbcr.cc", "ifb_pixel_convert.cc")   # of tests.cpu_emu.build
CTA_UNITS, RUN = 1024, 8                                                                            # ifb::kYeCtaUnits, kYeRun
MATTES = [(255, 255, 255, 255), (40, 200, 90, 255), (0, 0, 0, 0), (10, 120, 250, 128)]
_TABLES = []


def tables():
    """the library's t_lin and lut16k, which the kernel's matte reads (the CPU oracle of apply_matte holds the same values)"""
    if not _TABLES:
        import imageflow_b200 as ifb
        from tests import cpu_emu
        t_lin, _, lut = cpu_emu.transfer_tables(ifb)
        _TABLES.extend([t_lin, lut])
    return _TABLES


def load(so):
    L = C.CDLL(so)
    L.emu_bgra_to_ycbcr.restype = C.c_long
    L.emu_bgra_to_ycbcr.argtypes = [C.POINTER(BgraToYcbcrDesc), C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.c_char_p,
                                    C.c_size_t, C.c_int]
    L.emu_bgra_to_ycbcr_plan.restype = C.c_long
    L.emu_bgra_to_ycbcr_plan.argtypes = [C.POINTER(BgraToYcbcrDesc), C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p, C.c_size_t]
    return L


def make_job(rng, sampling=None, w=None, h=None, sphase=None, phases=None, matte=None, src=None, pitch16=False):
    """-> (desc dict, [Rows], {allowed load addresses}, {wanted store addresses}); `exp` of the plane Rows holds the result.
    sphase: the source's first-byte phase modulo 16 (a multiple of 4); phases: the Y, Cb and Cr planes' phases; matte: None (opaque)
    or a matte_bgra; src: a (h, w, 4) BGRA array to convert instead of the sentinel bytes; pitch16: every pitch a multiple of 16, so
    that every row starts at the phase of the first."""
    sampling = int(rng.choice(eo.SAMPLINGS)) if sampling is None else sampling
    w = (int(rng.integers(1, 41)) if w is None else w) if src is None else src.shape[1]
    h = (int(rng.integers(1, 7)) if h is None else h) if src is None else src.shape[0]
    sphase = 4 * int(rng.integers(0, 4)) if sphase is None else sphase
    phases = [int(p) for p in rng.integers(0, 16, 3)] if phases is None else phases
    ch, cw = eo.chroma_shape(sampling, w, h)

    def rows(w_, h_, ch_, phase):
        return Rows(rng, w_, h_, ch_, phase, -(-w_ * ch_ // 16) * 16) if pitch16 else rows_in(rng, w_, h_, ch_, phase, align4=ch_ == 4)
    s = rows(w, h, 4, sphase)
    if src is not None:
        s.view(s.buf)[...] = src
    elif matte is not None:                                     # alpha 0, 255 and values between
        a = s.view(s.buf)[..., 3]
        a[rng.random(a.shape) < 0.25] = 0
        a[rng.random(a.shape) < 0.25] = 255
    s.exp[:] = s.buf
    py, pb, pr = rows(w, h, 1, phases[0]), rows(cw, ch, 1, phases[1]), rows(cw, ch, 1, phases[2])
    bgra = s.view(s.buf).copy()
    planes = eo.convert_matte(sampling, bgra, matte, True) if matte is not None else eo.convert(sampling, bgra)
    for r, p in zip((py, pb, pr), planes):
        r.view(r.exp)[..., 0] = p
    d = dict(sampling=sampling, src=s.ptr, src_stride=s.pitch, y=py.ptr, y_stride=py.pitch, cb=pb.ptr, cb_stride=pb.pitch, cr=pr.ptr,
             cr_stride=pr.pitch, w=w, h=h, alpha_meaningful=int(matte is not None), matte_bgra=tuple(matte or (255, 255, 255, 255)))
    return d, [s, py, pb, pr], s.addrs(), py.addrs() | pb.addrs() | pr.addrs()


def descs_of(jobs):
    arr = (BgraToYcbcrDesc * len(jobs))()
    for desc, (d, *_rest) in zip(arr, jobs):
        for k, v in d.items():
            if k == "matte_bgra":
                desc.matte_bgra[:] = v
            else:
                setattr(desc, k, v)
    return arr


def launch(L, jobs, sabotage=0):
    """runs one call of the jobs on the emulator; -> (ctas, [load (address << 8 | width)], [store ...], items, error)"""
    arr = descs_of(jobs)
    t_lin, lut = tables()
    cap = 8 * sum(r.buf.size for _, rs, _, _ in jobs for r in rs) + 64
    loads, stores = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    nl, ns, ni = C.c_size_t(), C.c_size_t(), C.c_size_t()
    err = C.create_string_buffer(256)
    ctas = L.emu_bgra_to_ycbcr(arr, len(jobs), t_lin.ctypes.data, lut.ctypes.data, loads.ctypes.data, stores.ctypes.data, cap,
                               C.byref(nl), C.byref(ns), C.byref(ni), err, 256, sabotage)
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
    assert len(set(st_addr)) == len(st_addr), "a plane byte stored twice"
    assert set(st_addr) == want_st, "stored bytes differ from the plane windows"
    assert set((ld >> 8).tolist()) <= allowed, "a load outside the source windows"
    for _, rs, _, _ in jobs:
        for r in rs:
            diff = np.nonzero(r.buf != r.exp)[0]
            assert diff.size == 0, ("bytes differ", diff[:4].tolist())


def fixed_launches(rng):
    """every sampling at every source phase and plane phase; widths 1..40 and heights 1..6; mattes; items whose CTA boundaries fall
    inside a band; all three samplings and several sizes in one call"""
    out = []
    for s in eo.SAMPLINGS:
        jobs = [make_job(rng, s, w=1 + (i * 7) % 40, h=1 + i % 6, sphase=4 * (i % 4), phases=[i % 16, (i * 5 + 3) % 16, (i * 11 + 7) % 16])
                for i in range(48)]
        out += [jobs[i:i + 8] for i in range(0, len(jobs), 8)]
        out.append([make_job(rng, s, w=w, h=h) for w in (1, 2, 3, 4, 5) for h in (1, 2, 3, 4)])
        out.append([make_job(rng, s, w=w, h=h, matte=m) for m in MATTES for w, h in ((9, 3), (16, 2), (33, 5))])
    for w in range(1, 41):                                      # every width, each sampling once, mixed in one call
        out.append([make_job(rng, s, w=w, h=1 + w % 5) for s in eo.SAMPLINGS])
    # several CTAs per item: 147 columns are 19 units per band, which does not divide CTA_UNITS, so boundaries fall inside a band --
    # at 4:2:0 between the units of one row pair; whole 16-byte-aligned runs take the 16-byte loads
    out.append([make_job(rng, s, w=147, h=2 * 57 + 1, sphase=0, phases=[0, 0, 0]) for s in eo.SAMPLINGS])
    return out


def run(so, n_launches=200, seed=1):
    L = load(so)
    rng = np.random.default_rng(seed)
    cases = 0
    randoms = [[make_job(rng, matte=MATTES[int(rng.integers(0, 4))] if rng.random() < 0.3 else None)
                for _ in range(int(rng.integers(1, 9)))] for _ in range(n_launches)]
    for it, jobs in enumerate(fixed_launches(rng) + randoms):
        ctas, ld, st, _, err = launch(L, jobs)
        assert not err, err
        try:
            check(jobs, ctas, ld, st)
        except AssertionError as e:
            raise AssertionError((it, [j[0] for j in jobs], e.args))
        cases += len(jobs)
    return cases


def access_widths(so, sampling, w=301, h=4, sphase=0, phases=(0, 0, 0), seed=3):
    """{width: count} of the loads and of the stores of one job whose rows all start at the phases given (each access counted once,
    not per byte)"""
    L = load(so)
    rng = np.random.default_rng(seed)
    jobs = [make_job(rng, sampling, w=w, h=h, sphase=sphase, phases=list(phases), pitch16=True)]
    ctas, ld, st, _, err = launch(L, jobs)
    assert not err, err
    count = lambda a: {int(k): int(v) // int(k) for k, v in zip(*np.unique(a & 0xff, return_counts=True))}
    return count(ld), count(st)


def sabotage_caught(so, kind, seed=2):
    """True when the checks above reject the launch whose plan was corrupted in way `kind` (ycbcr_enc_kernel_emu.cc)"""
    L = load(so)
    rng = np.random.default_rng(seed)
    jobs = [make_job(rng, s, w=33, h=5, matte=MATTES[1]) for s in eo.SAMPLINGS]
    ctas, ld, st, _, err = launch(L, jobs, sabotage=kind)
    assert not err, err
    try:
        check(jobs, ctas, ld, st)
    except AssertionError:
        return True
    return False


if __name__ == "__main__":
    print("cases bit-exact:", run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 200))
