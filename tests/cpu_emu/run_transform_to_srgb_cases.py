"""python -m tests.cpu_emu.run_transform_to_srgb_cases <libtransform_to_srgb_kernel_emu.so> [n_launches]: the emulated
transform_to_srgb_kernel (tests/cpu_emu/transform_to_srgb_kernel_emu.cc, with the product's planner) against tests/profile_oracle.py.
Also the body of the AddressSanitizer run (the test starts it in a subprocess with libasan preloaded), which then also plans every
truncation of every fixture profile and seeded corruptions of their tag tables.

Every launch holds several jobs with mixed profiles (matrix ICC, gray ICC, gAMA+cHRM, CICP, sRGB) and all five source formats (BGRA,
in place or not, RGB24, RGBA32, Gray8, GrayAlpha8).  Each window lies inside an exactly sized bitmap of sentinel bytes
(tests/cpu_emu/run_pixel_convert_cases.Rows): BGRA destinations at every 4-byte phase modulo 16, 1-, 2- and 3-byte rows at every byte
phase.  Per launch:
  - every bitmap equals the expected one: pixel_convert's conversion, then the oracle's transform (tests/profile_oracle.apply_plan) in
    the destination window; every other byte unchanged, and an sRGB job in place unchanged;
  - every destination byte is stored exactly once, and nothing else is stored;
  - every load lies in a source window;
  - the profiles planned are the distinct ones of the call, compared by their bytes (copies of one profile share a plan)."""
import ctypes as C
import sys

import numpy as np

import imageflow_b200 as ifb
from imageflow_b200._lib import SourceProfileDesc, ToSrgbDesc
from tests import pixel_convert_oracle as po
from tests import profile_oracle as pf
from tests.cpu_emu.run_pixel_convert_cases import rows_in

SOURCES = ("transform_to_srgb_kernel_emu.cc", "ifb_profile.cc", "ifb_pixel_convert.cc", "ifb_weights.cc")   # of tests.cpu_emu.build
BGRA = 16
FORMATS = (BGRA, po.RGB24_TO_BGRA, po.RGBA_TO_BGRA, po.GRAY_TO_BGRA, po.GRAY_ALPHA_TO_BGRA)
SRC_CHANNELS = {BGRA: 4, po.RGB24_TO_BGRA: 3, po.RGBA_TO_BGRA: 4, po.GRAY_TO_BGRA: 1, po.GRAY_ALPHA_TO_BGRA: 2}


def load(so):
    L = C.CDLL(so)
    L.emu_transform_to_srgb.restype = C.c_long
    L.emu_transform_to_srgb.argtypes = [C.POINTER(ToSrgbDesc), C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                        C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), C.POINTER(C.c_size_t),
                                        C.c_char_p, C.c_size_t]
    L.emu_profile_plan.restype = C.c_int
    L.emu_profile_plan.argtypes = [C.POINTER(SourceProfileDesc), C.c_char_p, C.c_size_t]
    return L


def profiles():
    """the profiles the launches mix: (name, SourceProfile)"""
    fx = pf.fixtures()
    out = [(n, ifb.SourceProfile.icc(b) if k == "icc" else ifb.SourceProfile.icc_gray(b)) for n, (k, b) in fx.items()]
    out += [("srgb", ifb.SourceProfile.srgb()), ("cicp_p3", ifb.SourceProfile.cicp(12, 13)), ("cicp_srgb", ifb.SourceProfile.cicp(1, 13)),
            ("gama_linear", ifb.SourceProfile.gamma_primaries(1.0, *pf.SRGB_XY))]
    return out


def lut16k():
    from tests import cpu_emu
    return cpu_emu.transfer_tables(ifb)[2]


def make_job(rng, prof, fmt=None, w=None, h=None, sphase=None, dphase=None, in_place=None, copy_bytes=False):
    """-> (desc dict, profile, [Rows], {allowed load addresses}, {wanted store addresses}); `exp` of the Rows holds the result"""
    name, p = prof
    if copy_bytes and p.icc_bytes:                                # same bytes at another address: must share the plan
        p = ifb.SourceProfile(p.kind, bytes(bytearray(p.icc_bytes)))
    fmt = int(rng.choice(FORMATS)) if fmt is None else fmt
    cs = SRC_CHANNELS[fmt]
    w = int(rng.integers(1, 41)) if w is None else w
    h = int(rng.integers(1, 5)) if h is None else h
    dphase = 4 * int(rng.integers(0, 4)) if dphase is None else dphase
    in_place = (fmt == BGRA and rng.random() < 0.4) if in_place is None else in_place
    plan = ifb.source_profile_plan(p)
    lut = LUT[0]
    if in_place:
        r = rows_in(rng, w, h, 4, dphase, align4=True)
        r.view(r.exp)[...] = pf.apply_plan(plan, lut, r.view(r.buf).copy())
        d = dict(format=fmt, src=r.ptr, src_stride=r.pitch, dst=r.ptr, dst_stride=r.pitch, w=w, h=h)
        return d, p, [r], r.addrs(), (set() if plan.kind == 0 else r.addrs())
    sphase = int(rng.integers(0, 16)) if sphase is None else sphase
    s = rows_in(rng, w, h, cs, sphase)
    t = rows_in(rng, w, h, 4, dphase, align4=True)
    src = s.view(s.buf).copy()
    bgra = src if fmt == BGRA else po.convert(fmt, src)
    t.view(t.exp)[...] = pf.apply_plan(plan, lut, bgra)
    d = dict(format=fmt, src=s.ptr, src_stride=s.pitch, dst=t.ptr, dst_stride=t.pitch, w=w, h=h)
    return d, p, [s, t], s.addrs(), t.addrs()


LUT = [None]


def launch(L, jobs):
    """runs one call of the jobs on the emulator; -> (ctas, loads, stores, items, plans, error)"""
    arr = (ToSrgbDesc * len(jobs))()
    pds = []
    for desc, (d, p, *_rest) in zip(arr, jobs):
        for k, v in d.items():
            setattr(desc, k, v)
        pds.append(p._desc())
        desc.profile = C.cast(C.byref(pds[-1]), C.c_void_p)
    cap = 2 * sum(r.buf.size for _, _, rs, _, _ in jobs for r in rs) + 64
    loads, stores = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    nl, ns, ni, npl = C.c_size_t(), C.c_size_t(), C.c_size_t(), C.c_size_t()
    err = C.create_string_buffer(512)
    ctas = L.emu_transform_to_srgb(arr, len(jobs), LUT[0].ctypes.data, loads.ctypes.data, stores.ctypes.data, cap, C.byref(nl), C.byref(ns),
                                   C.byref(ni), C.byref(npl), err, 512)
    assert nl.value <= cap and ns.value <= cap
    return ctas, loads[:nl.value], stores[:ns.value], ni.value, npl.value, err.value.decode()


def distinct_profiles(jobs):
    keys = set()
    for d, p, *_ in jobs:
        if d["w"] and d["h"]:
            keys.add((p.kind, p.icc_bytes, p.gamma, p.chrm, p.cicp_codes))
    return len(keys)


def check(jobs, ctas, ld, st, n_plans):
    assert ctas >= 0, ctas
    allowed, want_st = set(), set()
    for _, _, _, reads, writes in jobs:
        allowed |= reads
        want_st |= writes
    st_addr = (st >> 8).tolist()
    assert len(set(st_addr)) == len(st_addr), "a destination byte stored twice"
    assert set(st_addr) == want_st, "stored bytes differ from the destination windows"
    assert set((ld >> 8).tolist()) <= allowed, "a load outside the source windows"
    for _, _, rs, _, _ in jobs:
        for r in rs:
            diff = np.nonzero(r.buf != r.exp)[0]
            assert diff.size == 0, ("bytes differ", diff[:4].tolist())
    assert n_plans == distinct_profiles(jobs), (n_plans, distinct_profiles(jobs))


def fixed_launches(rng, profs):
    """every format at every source byte phase modulo 16 and every destination 4-byte phase, widths 1..40, profiles in turn"""
    out = []
    for fmt in FORMATS:
        jobs = [make_job(rng, profs[i % len(profs)], fmt, w=1 + (i * 7) % 40, h=1 + i % 3, sphase=i % 16, dphase=4 * (i % 4), in_place=False)
                for i in range(48)]
        out += [jobs[i:i + 8] for i in range(0, len(jobs), 8)]
    out.append([make_job(rng, profs[i % len(profs)], BGRA, w=w, dphase=4 * (i % 4), in_place=True)
                 for i, w in enumerate((1, 3, 4, 5, 8, 13, 17, 33) * 2)])
    # one profile many times, some as copies of its bytes at other addresses: planned once
    out.append([make_job(rng, profs[0], copy_bytes=i % 2 == 1) for i in range(12)])
    return out


def run(so, n_launches=60, seed=1):
    L = load(so)
    LUT[0] = lut16k()
    rng = np.random.default_rng(seed)
    profs = profiles()
    cases = 0
    randoms = [[make_job(rng, profs[int(rng.integers(0, len(profs)))]) for _ in range(int(rng.integers(1, 9)))] for _ in range(n_launches)]
    randoms.append([make_job(rng, profs[k % len(profs)], fmt, w=int(rng.integers(600, 1400)), h=int(rng.integers(6, 12)))
                    for k, fmt in enumerate(FORMATS)])
    for it, jobs in enumerate(fixed_launches(rng, profs) + randoms):
        ctas, ld, st, _, n_plans, err = launch(L, jobs)
        assert not err, err
        try:
            check(jobs, ctas, ld, st, n_plans)
        except AssertionError as e:
            raise AssertionError((it, [(j[0], j[1].kind) for j in jobs], e.args))
        cases += len(jobs)
    return cases


def plan_status(L, profile):
    """(status, why) of the product planner on an exactly sized copy of the profile's bytes"""
    why = C.create_string_buffer(512)
    d = profile._desc()
    return L.emu_profile_plan(C.byref(d), why, 512), why.value.decode()


def corruptions(data, rng, n):
    """n seeded corruptions of an ICC profile's tag count, tag offsets and sizes, curve counts and header size"""
    be = lambda b, o: int.from_bytes(b[o:o + 4], "big")
    ntags = be(data, 128)
    for _ in range(n):
        b = bytearray(data)
        what = int(rng.integers(0, 5))
        val = int(rng.choice([0, 1, 2, 3, 4, 11, 12, 19, 20, 127, 128, 131, 132, len(b) - 1, len(b), len(b) + 1, 0x7fffffff, 0xfffffff0,
                              0xffffffff, int(rng.integers(0, 1 << 32))]))
        if what == 0:
            b[128:132] = val.to_bytes(4, "big")
        elif what == 1 and ntags:
            o = 132 + 12 * int(rng.integers(0, ntags)) + 4 * int(rng.integers(1, 3))
            b[o:o + 4] = val.to_bytes(4, "big")
        elif what == 2:
            b[0:4] = val.to_bytes(4, "big")
        elif what == 3 and ntags:                                 # the count / function type inside a tag's data
            o = be(b, 132 + 12 * int(rng.integers(0, ntags)) + 4)
            if o + 12 <= len(b):
                b[o + 8:o + 12] = val.to_bytes(4, "big")
        else:
            o = int(rng.integers(0, len(b)))
            b[o] = int(rng.integers(0, 256))
        yield bytes(b)


def robustness(so, n_corrupt=10000, seed=7):
    """every truncation of every fixture and n_corrupt seeded corruptions, through the planner: each returns a status.  -> counts"""
    L = load(so)
    rng = np.random.default_rng(seed)
    counts = {}
    fx = list(pf.fixtures().items())
    for name, (kind, data) in fx:
        mk = ifb.SourceProfile.icc if kind == "icc" else ifb.SourceProfile.icc_gray
        for k in range(len(data)):
            code, _ = plan_status(L, mk(data[:k]))
            assert code in (1, 2), (name, k, code)
            counts[code] = counts.get(code, 0) + 1
    per = n_corrupt // len(fx) + 1
    for name, (kind, data) in fx:
        mk = ifb.SourceProfile.icc if kind == "icc" else ifb.SourceProfile.icc_gray
        for b in corruptions(data, rng, per):
            code, _ = plan_status(L, mk(b))
            assert code in (0, 1, 2), (name, code)
            counts[code] = counts.get(code, 0) + 1
    return counts


if __name__ == "__main__":
    print("cases bit-exact:", run(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else 60))
    print("plan statuses:", robustness(sys.argv[1]))
