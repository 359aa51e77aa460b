"""The host planner of the colour-profile transform (imageflow_b200/csrc/ifb_profile.cc, through ifb200_source_profile_plan; no GPU):
its tables and matrix against an independent float64 restatement (tests/profile_oracle.py), the profiles it refuses and why, its
robustness on truncated and corrupted ICC bytes, and the band that the fp32 arithmetic it feeds keeps from the float64 transform on
every RGB triple."""
import os

import numpy as np
import pytest

import imageflow_b200 as ifb
from imageflow_b200 import ErrorKind, FlowError, SourceProfile
from tests import profile_oracle as pf

GOLDEN_GRAY = os.path.join(os.path.dirname(__file__), "golden", "gray.icc")     # the reference's codecs/gray.icc (v2.4, 1024-entry kTRC)


def fixture_profiles():
    out = {n: (SourceProfile.icc(b) if k == "icc" else SourceProfile.icc_gray(b)) for n, (k, b) in pf.fixtures().items()}
    out["golden_gray"] = SourceProfile.icc_gray(open(GOLDEN_GRAY, "rb").read())
    return out


FIXTURES = fixture_profiles()


@pytest.fixture(scope="module")
def lut16k():
    from tests import cpu_emu
    return cpu_emu.transfer_tables(ifb)[2]


def assert_plan_matches_f64(profile, lut):
    plan = ifb.source_profile_plan(profile)
    r = pf.restate(profile)
    if r[0] == "gray":
        assert plan.kind == plan.GRAY
        t64 = pf.clip01(r[1](np.arange(256) / 255.0))
        got = plan.trc[0].astype(np.float64)
        assert (np.abs(got - t64) <= np.spacing(np.abs(t64).astype(np.float32)).astype(np.float64)).all()
        assert np.array_equal(plan.gray, pf.encode_f32(lut, plan.trc[0]))
        return plan
    trcs, m64 = r
    assert plan.kind == plan.MATRIX
    t64 = pf.tables_f64(trcs)
    ulp = np.spacing(t64.astype(np.float32)).astype(np.float64)
    assert (np.abs(plan.trc.astype(np.float64) - t64) <= ulp).all(), np.abs(plan.trc - t64).max()
    assert np.abs(plan.m.astype(np.float64) - m64).max() <= 1e-6, (plan.m, m64)
    return plan


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_fixture_plan_matches_the_float64_restatement(name, lut16k):
    assert_plan_matches_f64(FIXTURES[name], lut16k)


@pytest.mark.parametrize("gamma", [1.0, 0.5, 0.35, 0.45455])
@pytest.mark.parametrize("chrm", [pf.SRGB_XY, pf.P3_XY], ids=["srgb", "p3"])
def test_gamma_primaries_plan(gamma, chrm, lut16k):
    assert_plan_matches_f64(SourceProfile.gamma_primaries(gamma, *chrm), lut16k)


@pytest.mark.parametrize("cp,tc", [(12, 13), (9, 1), (1, 8), (11, 13), (22, 6), (4, 4), (5, 5), (7, 7), (10, 8), (8, 14)])
def test_cicp_plan(cp, tc, lut16k):
    assert_plan_matches_f64(SourceProfile.cicp(cp, tc), lut16k)


def test_srgb_kinds_plan_to_the_identity():
    assert ifb.source_profile_plan(SourceProfile.srgb()).kind == 0
    assert ifb.source_profile_plan(SourceProfile.cicp(1, 13)).kind == 0
    assert ifb.source_profile_plan(SourceProfile.cicp(1, 13, 9, False)).kind == 0        # source_profile.rs:56 looks at cp / tc only


def test_prophoto_is_d50_native_and_srgb_is_nearly_the_identity():
    m = ifb.source_profile_plan(FIXTURES["srgb_para3_v4"]).m
    assert np.abs(m - np.eye(3)).max() < 2e-3
    t = ifb.source_profile_plan(FIXTURES["prophoto_v2"]).trc
    assert np.allclose(t[0], (np.arange(256) / 255.0) ** (461 / 256), atol=1e-6)


def _with_tag(data, sig, blob):
    """the RGB fixture `data` rewritten with one more tag"""
    parsed = []
    import struct
    n = struct.unpack_from(">I", data, 128)[0]
    for i in range(n):
        s, o, ln = struct.unpack_from(">4sII", data, 132 + 12 * i)
        parsed.append((s, data[o:o + ln]))
    return pf.write_icc(data[16:20], parsed + [(sig, blob)], data[8], pcs=data[20:24])


P3 = pf.fixtures()["display_p3_v4"][1]
GRAY = pf.fixtures()["gray22_v2"][1]
REFUSALS = {
    "a2b0_tag": (SourceProfile.icc(_with_tag(P3, b"A2B0", b"mAB " + b"\0" * 28)), ErrorKind.MethodNotImplemented, "A2B0"),
    "b2a1_tag": (SourceProfile.icc(_with_tag(P3, b"B2A1", b"mft2" + b"\0" * 48)), ErrorKind.MethodNotImplemented, "B2A1"),
    "mft1_type": (SourceProfile.icc(_with_tag(P3, b"gamt", b"mft1" + b"\0" * 44)), ErrorKind.MethodNotImplemented, "mft1"),
    "mba_type": (SourceProfile.icc(_with_tag(P3, b"pre0", b"mBA " + b"\0" * 28)), ErrorKind.MethodNotImplemented, "mBA"),
    "lab_pcs": (SourceProfile.icc(pf.write_icc(b"RGB ", [(b"rTRC", pf.curv_tag([]))], 4, pcs=b"Lab ")), ErrorKind.MethodNotImplemented, "Lab"),
    "cmyk": (SourceProfile.icc(pf.lut_profile()), ErrorKind.MethodNotImplemented, "CMYK"),
    "cmyk_no_lut": (SourceProfile.icc(pf.write_icc(b"CMYK", [], 2)), ErrorKind.MethodNotImplemented, "CMYK"),
    "pq": (SourceProfile.cicp(9, 16), ErrorKind.MethodNotImplemented, "PQ"),
    "hlg": (SourceProfile.cicp(9, 18), ErrorKind.MethodNotImplemented, "HLG"),
    "unknown_transfer": (SourceProfile.cicp(1, 17), ErrorKind.MethodNotImplemented, "transfer"),
    "unknown_primaries": (SourceProfile.cicp(3, 13), ErrorKind.MethodNotImplemented, "primaries"),
    "narrow_range": (SourceProfile.cicp(12, 13, 0, False), ErrorKind.MethodNotImplemented, "narrow"),
    "mc_not_0": (SourceProfile.cicp(12, 13, 1, True), ErrorKind.MethodNotImplemented, "matrix coefficients"),
    "rgb_as_gray": (SourceProfile.icc_gray(P3), ErrorKind.InvalidArgument, "ICC_GRAY"),
    "gray_as_rgb": (SourceProfile.icc(GRAY), ErrorKind.InvalidArgument, "GRAY ICC profile given as ICC"),
    "truncated": (SourceProfile.icc(P3[:200]), ErrorKind.InvalidArgument, "truncated"),
    "no_acsp": (SourceProfile.icc(P3[:36] + b"xxxx" + P3[40:]), ErrorKind.InvalidArgument, "acsp"),
    "missing_trc": (SourceProfile.icc(pf.write_icc(b"RGB ", [(b"rXYZ", pf.xyz_tag((0.4, 0.2, 0.0)))], 4)), ErrorKind.InvalidArgument, "no rTRC tag"),
    "para_type_5": (SourceProfile.icc(pf.rgb_profile(pf.SRGB_XY, [pf.para_tag(5, (1, 1, 1, 1, 1, 1, 1, 1))] * 3)), ErrorKind.InvalidArgument, "function type"),
    "empty": (SourceProfile.icc(b""), ErrorKind.InvalidArgument, "ICC"),
    "gamma_zero": (SourceProfile.gamma_primaries(0.0, *pf.SRGB_XY), ErrorKind.InvalidArgument, "gAMA"),
    "degenerate_chrm": (SourceProfile.gamma_primaries(0.45, 0.3127, 0.329, 0.3, 0.3, 0.3, 0.3, 0.3, 0.3), ErrorKind.InvalidArgument, "cHRM"),
}


@pytest.mark.parametrize("name", sorted(REFUSALS))
def test_refusals_give_their_status_and_reason(name):
    profile, kind, why = REFUSALS[name]
    with pytest.raises(FlowError) as e:
        ifb.source_profile_plan(profile)
    assert e.value.kind == kind, (e.value.kind, str(e.value))
    assert why in str(e.value)


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_every_truncation_returns_a_status(name):
    data = FIXTURES[name].icc_bytes
    for k in range(len(data)):
        with pytest.raises(FlowError) as e:
            ifb.source_profile_plan(SourceProfile(FIXTURES[name].kind, data[:k]))
        assert e.value.kind == ErrorKind.InvalidArgument


def test_seeded_corruptions_return_a_status():
    from tests.cpu_emu.run_transform_to_srgb_cases import corruptions
    rng = np.random.default_rng(11)
    seen = set()
    for name, p in sorted(FIXTURES.items()):
        for b in corruptions(p.icc_bytes, rng, 10000 // len(FIXTURES) + 1):
            try:
                ifb.source_profile_plan(SourceProfile(p.kind, b))
                seen.add(0)
            except FlowError as e:
                assert e.kind in (ErrorKind.InvalidArgument, ErrorKind.MethodNotImplemented), e
                seen.add(int(e.kind))
    assert {0, 1} <= seen


# ---------------------------------------------------------------- the band: oracle vs float64 on all 2^24 triples
BAND_CHUNK = 1 << 21


@pytest.mark.parametrize("name", sorted(n for n in FIXTURES if FIXTURES[n].kind == SourceProfile.ICC))
def test_oracle_within_one_level_of_float64_on_every_triple(name, lut16k):
    profile = FIXTURES[name]
    plan = ifb.source_profile_plan(profile)
    trcs, m64 = pf.restate(profile)
    i = np.arange(1 << 24, dtype=np.uint32)
    worst, at_one, not_identity = 0, 0, 0
    for a in range(0, 1 << 24, BAND_CHUNK):
        k = i[a:a + BAND_CHUNK]
        b, g, r = (k & 255).astype(np.uint8), ((k >> 8) & 255).astype(np.uint8), (k >> 16).astype(np.uint8)
        bgra = np.stack([b, g, r, np.full_like(b, 255)], -1)
        got = pf.apply_plan(plan, lut16k, bgra)[:, :3].astype(np.int64)
        eb, eg, er = pf.exact_bgr(trcs, m64, b, g, r)
        d = np.abs(got - np.stack([eb, eg, er], -1)).max(axis=1)
        if d.max() > 1:
            bad = np.nonzero(d > 1)[0][:8]
            pytest.fail(f"{name}: triples off by more than 1 level (B, G, R): {[tuple(bgra[j, :3]) for j in bad]}")
        worst = max(worst, int(d.max()))
        at_one += int((d == 1).sum())
        not_identity += int((got != bgra[:, :3]).any(axis=1).sum())
    print(f"\n{name}: max |d| {worst}, triples at |d| = 1: {at_one}" +
          (f", triples that differ from the identity: {not_identity}" if name.startswith("srgb") else ""))


@pytest.mark.parametrize("name", sorted(n for n in FIXTURES if FIXTURES[n].kind == SourceProfile.ICC_GRAY))
def test_gray_oracle_within_one_level_of_float64(name, lut16k):
    plan = ifb.source_profile_plan(FIXTURES[name])
    _, trc = pf.restate(FIXTURES[name])
    d = np.abs(plan.gray.astype(np.int64) - pf.exact_gray(trc, np.arange(256)))
    assert d.max() <= 1, np.nonzero(d > 1)[0]
    print(f"\n{name}: max |d| {int(d.max())}, values at |d| = 1: {int((d == 1).sum())}")
