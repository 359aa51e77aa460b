"""The watermark kernels (imageflow_b200/csrc/ifb_watermark_kernel.cuh: vpass_f_kernel and watermark_composite_kernel, the product's
CUDA source) executed on the CPU under a sequential emulation of the CUDA built-ins they use, with the product's host planner
(ifb_watermark.cc) validating and planning the calls exactly as the engine does: multi-job calls that share watermarks, with every
opacity case, compose mode, format and working space, on sub-windows of exactly sized bitmaps of sentinel bytes at every 4-byte phase,
checked for F, for the results, for the pixels stored (each once), for the loads (only the job's rectangle and its group's F) and for
the bytes around the rectangles (tests/cpu_emu/run_watermark_cases.py); then the same under AddressSanitizer; and plans corrupted on
purpose, which the checks must reject.  The kernels also run on the GPU (tests/test_watermark_gpu.py)."""
import pytest

from tests import cpu_emu
from tests.cpu_emu import run_watermark_cases


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    return cpu_emu.build(str(tmp_path_factory.mktemp("watermark_emu")), *run_watermark_cases.SOURCES)


def test_emulated_watermark_kernels_match_the_node_by_node_expansion(emu_so):
    assert run_watermark_cases.run(emu_so, 60) >= 200


@pytest.mark.parametrize("kind", [1, 2, 3], ids=["wrong_f_offset", "rows_cut_short", "two_jobs_on_one_rectangle"])
def test_a_sabotaged_plan_is_caught(emu_so, kind):
    assert run_watermark_cases.sabotage_caught(emu_so, kind)


def test_an_unsabotaged_sabotage_case_passes(emu_so):
    assert not run_watermark_cases.sabotage_caught(emu_so, 0)


def test_emulated_watermark_kernels_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), *run_watermark_cases.SOURCES, sanitize=True)
    r = cpu_emu.run_under_asan("run_watermark_cases", so, 25)
    assert r.returncode == 0 and "cases bit-exact:" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
