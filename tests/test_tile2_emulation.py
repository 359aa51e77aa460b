"""fused_tile2_kernel (imageflow_b200/csrc/ifb_tile2_kernel.cuh, the product's CUDA source) executed on the CPU: one OS thread
per CUDA thread, std::barrier for __syncthreads (tests/cpu_emu/tile2_kernel_emu.cc).  (1) every result byte equals the oracle's;
(2) the same run under AddressSanitizer, with shared memory as an exactly-sized heap block: no access outside shared memory, the
bitmaps or the tables.  The kernel is also verified on the GPU (tests/test_gpu_parity.py); this is what lets a change to it be
checked -- results and memory accesses -- before any GPU time is spent."""
from tests import cpu_emu
from tests.cpu_emu import run_tile2_cases


def test_emulated_kernel_is_bit_exact(tmp_path):
    so = cpu_emu.build(str(tmp_path), "tile2_kernel_emu.cc")
    assert run_tile2_cases.run(so) >= 40


def test_emulated_kernel_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), "tile2_kernel_emu.cc", sanitize=True)
    r = cpu_emu.run_under_asan("run_tile2_cases", so, 10)
    assert r.returncode == 0 and "cases bit-exact: 10" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
