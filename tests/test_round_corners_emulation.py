"""round_corners_kernel (imageflow_b200/csrc/ifb_round_corners_kernel.cuh, the product's CUDA source) executed on the CPU under a
sequential emulation of the CUDA built-ins it uses, with the product's host planner (ifb_round_corners.cc) making the jobs and the
work list exactly as the engine does: multi-job launches of sub-windows with sentinel bytes, checked against the oracle for results,
for the set of pixels written (each by one thread only) and for the pixels read (tests/cpu_emu/run_round_corners_cases.py); then
the same under AddressSanitizer.  The kernel is also verified on the GPU (tests/test_round_corners_gpu.py)."""
import pytest

from tests import cpu_emu
from tests.cpu_emu import run_round_corners_cases


def test_emulated_round_corners_kernel_matches_the_oracle(tmp_path):
    so = cpu_emu.build(str(tmp_path), *run_round_corners_cases.SOURCES)
    assert run_round_corners_cases.run(so, 600) >= 2000


def test_emulated_round_corners_kernel_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), *run_round_corners_cases.SOURCES, sanitize=True)
    r = cpu_emu.run_under_asan("run_round_corners_cases", so, 150)
    assert r.returncode == 0 and "cases bit-exact:" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
