"""round_corners_kernel (imageflow_b200/csrc/ifb_round_corners_kernel.cuh, the product's CUDA source) executed on the CPU under a
sequential emulation of the CUDA built-ins it uses, with the product's host planner (ifb_round_corners.cc) making the jobs and the
work list exactly as the engine does: multi-job launches of sub-windows with sentinel bytes, checked against the oracle for results,
for the set of pixels written (each by one thread only) and for the pixels read (tests/cpu_emu/run_round_corners_cases.py); then
the same under AddressSanitizer.  The kernel is also verified on the GPU (tests/test_round_corners_gpu.py)."""
import os
import subprocess
import sys

import pytest

from tests.cpu_emu import run_round_corners_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_emulated_round_corners_kernel_matches_the_oracle(tmp_path):
    so = run_round_corners_cases.build(str(tmp_path))
    assert run_round_corners_cases.run(so, 600) >= 2000


def test_emulated_round_corners_kernel_under_address_sanitizer(tmp_path):
    asan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan) or not os.path.exists(asan):
        pytest.skip("libasan not available")
    so = run_round_corners_cases.build(str(tmp_path), sanitize=True)
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:verify_asan_link_order=0", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "tests.cpu_emu.run_round_corners_cases", so, "150"], capture_output=True, text=True, cwd=ROOT,
                       env=env, timeout=1200)
    assert r.returncode == 0 and "cases bit-exact:" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
