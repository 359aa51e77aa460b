"""pixel_convert_kernel (imageflow_b200/csrc/ifb_pixel_convert_kernel.cuh, the product's CUDA source) executed on the CPU under a
sequential emulation of the CUDA built-ins it uses, with the product's host planner (ifb_pixel_convert.cc) validating and planning the
calls exactly as the engine does: multi-job calls of all five ops on sub-windows of exactly sized bitmaps of sentinel bytes, at every
source byte phase and destination phase, checked for results, for the bytes stored (each once) and for the bytes loaded
(tests/cpu_emu/run_pixel_convert_cases.py); then the same under AddressSanitizer; and plans corrupted on purpose, which the checks must
reject.  The kernel is also run on the GPU (tests/test_pixel_convert_gpu.py)."""
import pytest

from tests import cpu_emu
from tests import pixel_convert_oracle as po
from tests.cpu_emu import run_pixel_convert_cases


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    return cpu_emu.build(str(tmp_path_factory.mktemp("pixel_convert_emu")), *run_pixel_convert_cases.SOURCES)


def test_emulated_pixel_convert_kernel_matches_the_oracle(emu_so):
    assert run_pixel_convert_cases.run(emu_so, 200) >= 1000


@pytest.mark.parametrize("op", po.OPS)
def test_only_the_ragged_ends_of_a_row_take_byte_loads(emu_so, op):
    """At a source phase that no word access fits, a row's interior still runs on word loads: byte loads are bounded per row, not
    per pixel."""
    words, bytes_, rows = run_pixel_convert_cases.narrow_accesses(emu_so, op, w=301, h=4, sphase=5)
    assert bytes_ <= 6 * rows and words >= 301 * 4 * po.CHANNELS[op][0] // 4 // 2


@pytest.mark.parametrize("kind", [1, 2, 3], ids=["wrong_first_cta", "rows_cut_short", "two_jobs_on_one_rectangle"])
def test_a_sabotaged_plan_is_caught(emu_so, kind):
    assert run_pixel_convert_cases.sabotage_caught(emu_so, kind)


def test_emulated_pixel_convert_kernel_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), *run_pixel_convert_cases.SOURCES, sanitize=True)
    r = cpu_emu.run_under_asan("run_pixel_convert_cases", so, 80)
    assert r.returncode == 0 and "cases bit-exact:" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
