"""hv_ring_kernel (imageflow_b200/csrc/ifb_hv_kernel.cuh, the product's CUDA source of the hot kernel) executed on the CPU: one OS
thread per CUDA thread, per-warp barriers behind the warp-synchronous primitives, the TMA box load emulated with the hardware's
SWIZZLE_64B address transform, the mbarrier phases checked (tests/cpu_emu/hv_kernel_emu.cc), over the host tables the engine
would upload (ifb200_hv_plan_tables).  (1) every result byte equals the oracle's, for both ring depths, both channel counts, every
compositing mode, strips, bands, unaligned window origins and another shared-memory origin; (2) the same run under
AddressSanitizer with shared memory as an exactly-sized heap block.  The kernel is also verified on the GPU
(tests/test_gpu_parity.py); this is what lets a change to it be checked -- results, barrier phases, memory accesses -- before any
GPU time is spent."""
from tests import cpu_emu
from tests.cpu_emu import run_hv_cases


def test_emulated_hv_kernel_is_bit_exact(tmp_path):
    so = cpu_emu.build(str(tmp_path), "hv_kernel_emu.cc")
    assert run_hv_cases.run(so) >= 20


def test_emulated_hv_kernel_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), "hv_kernel_emu.cc", sanitize=True)
    r = cpu_emu.run_under_asan("run_hv_cases", so, 5)
    assert r.returncode == 0 and "cases bit-exact: 5" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
