"""The colour-chain kernels (imageflow_b200/csrc/ifb_color_kernel.cuh, the product's CUDA source) executed on the CPU under a
sequential emulation of the CUDA built-ins they use, with the product's host planner (ifb_color.cc) validating and planning the calls
exactly as the engine does: multi-job calls of random chains, with and without white balance, on sub-windows of exactly sized bitmaps
of sentinel bytes at every 4-byte phase modulo 16, checked for results, for the pixels stored (each once), for the pixels loaded and
for the white balance's histograms (tests/cpu_emu/run_color_cases.py); then the same under AddressSanitizer; and plans corrupted on
purpose, which the checks must reject.  The kernels are also run on the GPU (tests/test_color_chain_gpu.py)."""
import pytest

from tests import cpu_emu
from tests.cpu_emu import run_color_cases


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    return cpu_emu.build(str(tmp_path_factory.mktemp("color_emu")), *run_color_cases.SOURCES)


def test_emulated_color_kernels_match_the_node_by_node_chain(emu_so):
    assert run_color_cases.run(emu_so, 200) >= 800


@pytest.mark.parametrize("kind", [1, 2, 3], ids=["tile_crosses_a_job", "wrong_table_offset", "white_balance_on_other_counters"])
def test_a_sabotaged_plan_is_caught(emu_so, kind):
    assert run_color_cases.sabotage_caught(emu_so, kind)


def test_emulated_color_kernels_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), *run_color_cases.SOURCES, sanitize=True)
    r = cpu_emu.run_under_asan("run_color_cases", so, 80)
    assert r.returncode == 0 and "cases bit-exact:" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
