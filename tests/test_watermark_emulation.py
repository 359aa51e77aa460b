"""The watermark kernels (imageflow_b200/csrc/ifb_watermark_kernel.cuh: vpass_f_kernel and watermark_composite_kernel, the product's
CUDA source) executed on the CPU under a sequential emulation of the CUDA built-ins they use, with the product's host planner
(ifb_watermark.cc) validating and planning the calls exactly as the engine does: multi-job calls that share watermarks, with every
opacity case, compose mode, format and working space, on sub-windows of exactly sized bitmaps of sentinel bytes at every 4-byte phase,
checked for F, for the results, for the pixels stored (each once), for the loads (only the job's rectangle and its group's F) and for
the bytes around the rectangles (tests/cpu_emu/run_watermark_cases.py); then the same under AddressSanitizer; and plans corrupted on
purpose, which the checks must reject.  The kernels also run on the GPU (tests/test_watermark_gpu.py)."""
import os
import subprocess
import sys

import pytest

from tests.cpu_emu import run_watermark_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    return run_watermark_cases.build(str(tmp_path_factory.mktemp("watermark_emu")))


def test_emulated_watermark_kernels_match_the_node_by_node_expansion(emu_so):
    assert run_watermark_cases.run(emu_so, 60) >= 200


@pytest.mark.parametrize("kind", [1, 2, 3], ids=["wrong_f_offset", "rows_cut_short", "two_jobs_on_one_rectangle"])
def test_a_sabotaged_plan_is_caught(emu_so, kind):
    assert run_watermark_cases.sabotage_caught(emu_so, kind)


def test_an_unsabotaged_sabotage_case_passes(emu_so):
    assert not run_watermark_cases.sabotage_caught(emu_so, 0)


def test_emulated_watermark_kernels_under_address_sanitizer(tmp_path):
    asan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan) or not os.path.exists(asan):
        pytest.skip("libasan not available")
    so = run_watermark_cases.build(str(tmp_path), sanitize=True)
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:verify_asan_link_order=0", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "tests.cpu_emu.run_watermark_cases", so, "25"], capture_output=True, text=True, cwd=ROOT,
                       env=env, timeout=1200)
    assert r.returncode == 0 and "cases bit-exact:" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
