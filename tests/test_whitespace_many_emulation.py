"""whitespace_segments_kernel and whitespace_walk_kernel (imageflow_b200/csrc/ifb_whitespace_kernel.cuh, the product's CUDA source)
executed on the CPU, with the product's host planner (ifb_whitespace.cc) validating and planning each call exactly as the engine
does: multi-frame calls over the _images corpora of tests/test_whitespace_product.py and the planner's geometries, at thresholds 0, 1,
80 and 255 and both alpha modes, rectangle and visited count equal to oracle.detect_content, sentinels around the summaries intact,
and no window whose columns would depend on the box (tests/cpu_emu/run_whitespace_many_cases.py); then the same under
AddressSanitizer.  The kernels are also run on the GPU (tests/test_whitespace_many_gpu.py)."""
from tests import cpu_emu
from tests.cpu_emu import run_whitespace_many_cases


def test_emulated_kernels_match_the_oracle(tmp_path):
    so = cpu_emu.build(str(tmp_path), *run_whitespace_many_cases.SOURCES)
    assert run_whitespace_many_cases.run(so) >= 1250


def test_emulated_kernels_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), *run_whitespace_many_cases.SOURCES, sanitize=True)
    r = cpu_emu.run_under_asan("run_whitespace_many_cases", so, 40)
    assert r.returncode == 0 and "cases exact:" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
