"""orient_kernel (imageflow_b200/csrc/ifb_orient_kernel.cuh, the product's CUDA source) executed on the CPU under a sequential
emulation of the CUDA built-ins it uses, with the product's host planner (ifb_orient.cc) validating and planning the calls exactly as
the engine does: multi-job calls of all eight flags, in place and out of place, on sub-windows of exactly sized bitmaps of sentinel
bytes, checked for results, for the pixels stored (each once), for the pixels loaded and for shared-memory indices
(tests/cpu_emu/run_orient_cases.py); then the same under AddressSanitizer; and plans corrupted on purpose, which the checks must
reject.  The kernel is also run on the GPU (tests/test_orient_gpu.py)."""
import os
import subprocess
import sys

import pytest

from tests.cpu_emu import run_orient_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    return run_orient_cases.build(str(tmp_path_factory.mktemp("orient_emu")))


def test_emulated_orient_kernel_matches_the_closed_form(emu_so):
    assert run_orient_cases.run(emu_so, 300) >= 1400


@pytest.mark.parametrize("kind", [1, 2, 3], ids=["x_reversal_toggled", "output_moved", "cta_dropped"])
def test_a_sabotaged_plan_is_caught(emu_so, kind):
    assert run_orient_cases.sabotage_caught(emu_so, kind)


def test_emulated_orient_kernel_under_address_sanitizer(tmp_path):
    asan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan) or not os.path.exists(asan):
        pytest.skip("libasan not available")
    so = run_orient_cases.build(str(tmp_path), sanitize=True)
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:verify_asan_link_order=0", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "tests.cpu_emu.run_orient_cases", so, "120"], capture_output=True, text=True, cwd=ROOT,
                       env=env, timeout=1200)
    assert r.returncode == 0 and "cases bit-exact:" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
