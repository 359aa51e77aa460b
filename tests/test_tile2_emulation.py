"""fused_tile2_kernel (imageflow_b200/csrc/ifb_tile2_kernel.cuh, the product's CUDA source) executed on the CPU: one OS thread
per CUDA thread, std::barrier for __syncthreads (tests/cpu_emu/tile2_kernel_emu.cc).  (1) every result byte equals the oracle's;
(2) the same run under AddressSanitizer, with shared memory as an exactly-sized heap block: no access outside shared memory, the
bitmaps or the tables.  The kernel is also verified on the GPU (tests/test_gpu_parity.py); this is what lets a change to it be
checked -- results and memory accesses -- before any GPU time is spent."""
import os
import subprocess
import sys

import pytest

from tests import cpu_emu
from tests.cpu_emu import run_tile2_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_emulated_kernel_is_bit_exact(tmp_path):
    so = cpu_emu.build_tile2(str(tmp_path))
    assert run_tile2_cases.run(so) >= 40


def test_emulated_kernel_under_address_sanitizer(tmp_path):
    asan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan) or not os.path.exists(asan):
        pytest.skip("libasan not available")
    so = cpu_emu.build_tile2(str(tmp_path), sanitize=True)
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0:verify_asan_link_order=0", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "tests.cpu_emu.run_tile2_cases", so, "10"], capture_output=True, text=True, cwd=ROOT, env=env, timeout=1200)
    assert r.returncode == 0 and "cases bit-exact: 10" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
