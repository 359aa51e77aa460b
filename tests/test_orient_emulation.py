"""orient_kernel (imageflow_b200/csrc/ifb_orient_kernel.cuh, the product's CUDA source) executed on the CPU under a sequential
emulation of the CUDA built-ins it uses, with the product's host planner (ifb_orient.cc) validating and planning the calls exactly as
the engine does: multi-job calls of all eight flags, in place and out of place, on sub-windows of exactly sized bitmaps of sentinel
bytes, checked for results, for the pixels stored (each once), for the pixels loaded and for shared-memory indices
(tests/cpu_emu/run_orient_cases.py); then the same under AddressSanitizer; and plans corrupted on purpose, which the checks must
reject.  The kernel is also run on the GPU (tests/test_orient_gpu.py)."""
import pytest

from tests import cpu_emu
from tests.cpu_emu import run_orient_cases


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    return cpu_emu.build(str(tmp_path_factory.mktemp("orient_emu")), *run_orient_cases.SOURCES)


def test_emulated_orient_kernel_matches_the_closed_form(emu_so):
    assert run_orient_cases.run(emu_so, 300) >= 1400


@pytest.mark.parametrize("kind", [1, 2, 3], ids=["x_reversal_toggled", "output_moved", "cta_dropped"])
def test_a_sabotaged_plan_is_caught(emu_so, kind):
    assert run_orient_cases.sabotage_caught(emu_so, kind)


def test_emulated_orient_kernel_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), *run_orient_cases.SOURCES, sanitize=True)
    r = cpu_emu.run_under_asan("run_orient_cases", so, 120)
    assert r.returncode == 0 and "cases bit-exact:" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
