"""canvas_kernel (imageflow_b200/csrc/ifb_canvas_kernel.cuh, the product's CUDA source) executed on the CPU under a sequential
emulation of the CUDA built-ins it uses, with the product's host planner (ifb_canvas.cc) validating and planning the calls exactly
as the engine does: multi-job calls mixing all four ops in exactly sized bitmaps of sentinel bytes, checked against the numpy oracle
for results, for the set of pixels written (each once) and for the pixels read (tests/cpu_emu/run_canvas_cases.py); then the same
under AddressSanitizer; and plans corrupted on purpose, which the checks must reject.  The kernel is also run on the GPU
(tests/test_canvas_gpu.py)."""
import pytest

from tests import cpu_emu
from tests.cpu_emu import run_canvas_cases


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    return cpu_emu.build(str(tmp_path_factory.mktemp("canvas_emu")), *run_canvas_cases.SOURCES)


def test_emulated_canvas_kernel_matches_the_oracle(emu_so):
    assert run_canvas_cases.run(emu_so, 400) >= 1500


@pytest.mark.parametrize("kind", [1, 2, 3], ids=["tile_run_twice", "item_moved", "tile_dropped"])
def test_a_sabotaged_plan_is_caught(emu_so, kind):
    assert run_canvas_cases.sabotage_caught(emu_so, kind)


def test_emulated_canvas_kernel_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), *run_canvas_cases.SOURCES, sanitize=True)
    r = cpu_emu.run_under_asan("run_canvas_cases", so, 150)
    assert r.returncode == 0 and "cases bit-exact:" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
