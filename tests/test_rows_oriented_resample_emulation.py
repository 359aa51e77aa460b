"""The oriented row-format forms of hv_ring_kernel (ifb_hv_kernel.cuh, ORI = HV_ORI_FLIP / HV_ORI_TRANSPOSE with SRC = HV_SRC_RGBA /
HV_SRC_RGB24: RGBA32 through the BGRA oriented boxes with blue and red swapped in the look-ups; RGB24 flips through 64-byte boxes
walked from the far end, RGB24 transposes through 128-byte x 16-row boxes) executed on the CPU by their emulator
(tests/cpu_emu/hv_rows_oriented_kernel_emu.cc: the product's source, all four tensor maps emulated with zero fill, box origins
checked to be 16-byte aligned, mbarrier phases checked), over the tables ifb200_hv_plan_tables gives for the oriented geometry.  Every
byte equals the oracle's scale_and_render of the rows converted to BGRA and oriented in numpy, for flags 2..8 and both formats, both
ring depths and channel counts, every compositing mode, colour matrices, sharpen, strips, bands, every byte phase of RGB24 rows mod
16 under reversed and transposed reads, widths that are not a multiple of four and sizes below one box; and the same run passes under
AddressSanitizer with the rows in a buffer that ends at the last row's last byte."""
from tests import cpu_emu
from tests.cpu_emu import run_rows_oriented_hv_cases



def test_emulated_oriented_rows_ring_kernel_is_bit_exact(tmp_path):
    so = cpu_emu.build(str(tmp_path), "hv_rows_oriented_kernel_emu.cc")
    assert run_rows_oriented_hv_cases.run(so) >= 100


def test_emulated_oriented_rows_ring_kernel_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), "hv_rows_oriented_kernel_emu.cc", sanitize=True)
    r = cpu_emu.run_under_asan("run_rows_oriented_hv_cases", so, 24)
    assert r.returncode == 0 and "oriented rows cases bit-exact: 24" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
