"""transform_to_srgb_kernel (imageflow_b200/csrc/ifb_profile_kernel.cuh, the product's CUDA source) executed on the CPU under a
sequential emulation of the CUDA built-ins it uses, with the product's host planner (ifb_profile.cc) validating and planning the calls
exactly as the engine does: multi-job calls with mixed profiles and all five source formats on sub-windows of exactly sized bitmaps of
sentinel bytes, checked for results, for the bytes stored (each once), for the bytes loaded and for the plans shared
(tests/cpu_emu/run_transform_to_srgb_cases.py); then the same, and the planner on every truncation and 10 000 corruptions of the
fixture profiles, under AddressSanitizer.  The kernel is also run on the GPU (tests/test_color_profile_gpu.py)."""
import pytest

from tests import cpu_emu
from tests.cpu_emu import run_transform_to_srgb_cases as cases


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    return cpu_emu.build(str(tmp_path_factory.mktemp("transform_to_srgb_emu")), *cases.SOURCES)


def test_emulated_transform_to_srgb_kernel_matches_the_oracle(emu_so):
    assert cases.run(emu_so, 60) >= 300


def test_emulated_planner_survives_truncations_and_corruptions(emu_so):
    counts = cases.robustness(emu_so, 2000)
    assert counts.get(1, 0) > 0 and set(counts) <= {0, 1, 2}


def test_emulated_transform_to_srgb_kernel_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), *cases.SOURCES, sanitize=True)
    r = cpu_emu.run_under_asan("run_transform_to_srgb_cases", so, 20)
    assert r.returncode == 0 and "cases bit-exact:" in r.stdout and "plan statuses:" in r.stdout and "AddressSanitizer" not in r.stderr, \
        (r.stdout[-300:], r.stderr[-1500:])
