"""The row-format forms of hv_ring_kernel (ifb_hv_kernel.cuh: RGBA32 through the BGRA box with blue and red swapped in the look-ups,
RGB24 through a UINT8 tensor in 64-byte boxes) executed on the CPU by their emulator (tests/cpu_emu/hv_rows_kernel_emu.cc: the
product's source, both tensor maps emulated with zero fill, box origins checked to be 16-byte aligned, mbarrier phases checked),
over the tables ifb200_hv_plan_tables gives.  Every byte equals the oracle's scale_and_render of the rows converted to BGRA in numpy,
for both formats, both ring depths and channel counts, every compositing mode, colour matrices, sharpen, strips, bands, every byte
phase of RGB24 rows mod 16, widths whose 3 in_w is and is not a multiple of 16 and sizes below one box; and the same run passes under
AddressSanitizer with the rows in a buffer that ends at the last row's last byte."""
from tests import cpu_emu
from tests.cpu_emu import run_rows_hv_cases


def test_emulated_rows_ring_kernel_is_bit_exact(tmp_path):
    so = cpu_emu.build(str(tmp_path), "hv_rows_kernel_emu.cc")
    assert run_rows_hv_cases.run(so) >= 30


def test_emulated_rows_ring_kernel_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), "hv_rows_kernel_emu.cc", sanitize=True)
    r = cpu_emu.run_under_asan("run_rows_hv_cases", so, 34)
    assert r.returncode == 0 and "rows cases bit-exact: 34" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
