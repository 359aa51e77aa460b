"""ycbcr_to_bgra_kernel (imageflow_b200/csrc/ifb_ycbcr_kernel.cuh, the product's CUDA source) executed on the CPU under a sequential
emulation of the CUDA built-ins it uses, with the product's host planner (ifb_ycbcr.cc) validating and planning the calls exactly as
the engine does: multi-job calls of all three samplings on planes and destinations inside exactly sized bitmaps of sentinel bytes, at
every plane byte phase and destination phase, with padded strides, items whose CTA boundaries fall inside a 4:2:0 row pair, and mixed
samplings and sizes in one call -- checked for results against tests/ycbcr_oracle.py, for the bytes stored (each once) and for the
bytes loaded (tests/cpu_emu/run_ycbcr_cases.py); then the same under AddressSanitizer, where an overrun of the halo reads at a plane's
edges would show; the libjpeg-turbo fixture through the kernel; and plans corrupted on purpose, which the checks must reject.  The
kernel is also run on the GPU (tests/test_ycbcr_gpu.py)."""
import numpy as np
import pytest

from tests import cpu_emu
from tests import ycbcr_oracle as yo
from tests.cpu_emu import run_pixel_convert_cases as rpc
from tests.cpu_emu import run_ycbcr_cases
from tests.test_ycbcr_oracle import CASES, golden_case


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    return cpu_emu.build(str(tmp_path_factory.mktemp("ycbcr_emu")), *run_ycbcr_cases.SOURCES)


def test_emulated_ycbcr_kernel_matches_the_oracle(emu_so):
    assert run_ycbcr_cases.run(emu_so, 200) >= 1000


def test_the_libjpeg_turbo_fixture_through_the_emulated_kernel(emu_so):
    """every golden case in one call, each plane and destination at an odd phase inside a bitmap of sentinel bytes"""
    L = run_ycbcr_cases.load(emu_so)
    rng = np.random.default_rng(5)
    jobs = []
    for i, name in enumerate(CASES):
        s, y, cb, cr, want = golden_case(name)
        h, w = y.shape
        rows = []
        for p, phase in zip((y, cb, cr), (i % 16, (i + 5) % 16, (i + 9) % 16)):
            r = rpc.rows_in(rng, p.shape[1], p.shape[0], 1, phase)
            r.view(r.buf)[..., 0] = p
            r.exp[:] = r.buf
            rows.append(r)
        t = rpc.rows_in(rng, w, h, 4, 4 * (i % 4), align4=True)
        t.view(t.exp)[...] = want
        d = dict(sampling=s, y=rows[0].ptr, y_stride=rows[0].pitch, cb=rows[1].ptr, cb_stride=rows[1].pitch, cr=rows[2].ptr,
                 cr_stride=rows[2].pitch, dst=t.ptr, dst_stride=t.pitch, w=w, h=h)
        jobs.append((d, rows + [t], set().union(*(r.addrs() for r in rows)), t.addrs()))
    ctas, ld, st, n_items, err = run_ycbcr_cases.launch(L, jobs)
    assert not err and n_items == len(CASES)
    run_ycbcr_cases.check(jobs, ctas, ld, st)


@pytest.mark.parametrize("sampling", yo.SAMPLINGS)
def test_only_the_ragged_ends_of_a_row_take_byte_loads(emu_so, sampling):
    """At plane phases that no word access fits, a row's interior still runs on word loads: byte loads are bounded per row (the ends
    of the luma row and of the chroma rows each unit reads), not per pixel."""
    for w in (301, 1201):
        words, bytes_, rows = run_ycbcr_cases.narrow_accesses(emu_so, sampling, w=w, h=4, phases=(5, 3, 7))
        assert bytes_ <= 32 * rows and words >= w * rows, (w, words, bytes_)


@pytest.mark.parametrize("kind", [1, 2, 3], ids=["wrong_first_cta", "rows_cut_short", "wrong_chroma_plane"])
def test_a_sabotaged_plan_is_caught(emu_so, kind):
    assert run_ycbcr_cases.sabotage_caught(emu_so, kind)


def test_emulated_ycbcr_kernel_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), *run_ycbcr_cases.SOURCES, sanitize=True)
    r = cpu_emu.run_under_asan("run_ycbcr_cases", so, 80)
    assert r.returncode == 0 and "cases bit-exact:" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
