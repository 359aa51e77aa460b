"""The profiled forms of the ring kernel (hv_ring_profiled_kernel, ifb_hv_kernel.cuh: a profile's plan applied to every source pixel
before the byte-to-float look-ups, its tables staged next to the flag word) executed on the CPU by their emulator
(tests/cpu_emu/hv_profiled_kernel_emu.cc: the product's source, all four tensor maps emulated with zero fill, box origins checked to
be 16-byte aligned, mbarrier phases checked).  Every byte equals the oracle chain (profile_oracle.apply_plan, orient_oracle.gather,
oracle.scale_and_render) for matrix and gray plans, flags 1..8, BGRA, RGBA32 and RGB24 sources with RGB24 at every byte phase, both
ring depths and channel counts, both simple store epilogues, sharpen, strips and bands; the first 45 runs, which reach both ring
depths, both channel counts, all three sources and both plans, pass under AddressSanitizer.  Host only: ifb::ProfilePlans shares one plan between
identical profiles, and transform_to_srgb_prepare, which plans through it, gives the same plans as before."""
import ctypes as C

import numpy as np
import pytest

from tests import cpu_emu, profile_oracle as pf
from tests.cpu_emu import run_profiled_hv_cases as cases

SOURCES = ("hv_profiled_kernel_emu.cc", "ifb_profile.cc", "ifb_pixel_convert.cc", "ifb_weights.cc")


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    return cpu_emu.build(str(tmp_path_factory.mktemp("hv_profiled_emu")), *SOURCES)


def test_emulated_profiled_ring_kernel_is_bit_exact(emu_so):
    n, reached = cases.run(emu_so)
    assert n >= 100
    assert {av for av, _, _, _ in reached} == {4, 6} and {ch for _, ch, _, _ in reached} == {3, 4}
    assert {f for _, _, f, _ in reached} == {"bgra", "rgba", "rgb24"} and {k for _, _, _, k in reached} == {1, 2}


def test_emulated_profiled_ring_kernel_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), *SOURCES, sanitize=True)
    r = cpu_emu.run_under_asan("run_profiled_hv_cases", so, 45)
    assert r.returncode == 0 and "profiled cases bit-exact: 45" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])


def _profiles(ifb):
    fx = pf.fixtures()
    def icc(n):
        kind, data = fx[n]
        return ifb.SourceProfile.icc(data) if kind == "icc" else ifb.SourceProfile.icc_gray(data)
    return [icc("display_p3_v4"), icc("adobe_rgb_v2"), icc("display_p3_v4"), ifb.SourceProfile.srgb(), icc("gray22_v2"),
            ifb.SourceProfile.cicp(9, 1), icc("adobe_rgb_v2"), ifb.SourceProfile.cicp(9, 1), ifb.SourceProfile.srgb()]


def _ptrs(profs):
    descs = [p._desc() for p in profs]
    arr = (C.c_void_p * len(descs))(*[C.addressof(d) for d in descs])
    return descs, arr


def test_profile_plans_share_identical_profiles_and_match_transform_to_srgb(emu_so):
    import imageflow_b200 as ifb
    L = C.CDLL(emu_so)
    profs = _profiles(ifb)
    keep, arr = _ptrs(profs)
    n = len(profs)
    plan_of, kinds, why = (C.c_uint32 * n)(), (C.c_int32 * n)(), C.create_string_buffer(256)
    k = L.emu_profile_plans(arr, C.c_size_t(n), plan_of, kinds, why, C.c_size_t(256))
    assert k == 5, why.value
    assert list(plan_of) == [0, 1, 0, 2, 3, 4, 1, 4, 2]
    assert list(kinds)[:k] == [ifb.source_profile_plan(profs[i]).kind for i in (0, 1, 3, 4, 5)] == [1, 1, 0, 2, 1]
    t_of = (C.c_uint32 * n)()
    assert L.emu_transform_plan_of(arr, C.c_size_t(n), t_of, why, C.c_size_t(256)) == 5, why.value
    assert list(t_of) == list(plan_of)


def test_profile_plans_report_the_first_refused_profile(emu_so):
    import imageflow_b200 as ifb
    L = C.CDLL(emu_so)
    profs = [ifb.SourceProfile.cicp(9, 1), ifb.SourceProfile.icc(pf.lut_profile()), ifb.SourceProfile.cicp(9, 16)]
    keep, arr = _ptrs(profs)
    plan_of, kinds, why = (C.c_uint32 * 3)(), (C.c_int32 * 3)(), C.create_string_buffer(256)
    assert L.emu_profile_plans(arr, C.c_size_t(3), plan_of, kinds, why, C.c_size_t(256)) == -2
    assert b"CMYK" in why.value
    assert L.emu_transform_plan_of(arr, C.c_size_t(3), plan_of, why, C.c_size_t(256)) == -1
    assert why.value.startswith(b"transform to srgb job 1: ") and b"CMYK" in why.value
