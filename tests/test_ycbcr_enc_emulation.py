"""bgra_to_ycbcr_kernel (imageflow_b200/csrc/ifb_ycbcr_enc_kernel.cuh, the product's CUDA source) executed on the CPU under a sequential
emulation of the CUDA built-ins it uses, with the product's host planner (ifb_ycbcr_enc.cc) validating and planning the calls exactly
as the engine does: multi-job calls of all three samplings from sources and into planes inside exactly sized bitmaps of sentinel bytes,
at every source and plane byte phase, with padded strides, items whose CTA boundaries fall inside a 4:2:0 row pair, mattes, and mixed
samplings and sizes in one call -- checked for results against tests/ycbcr_enc_oracle.py (every sample asserted to need no clamp), for
the bytes stored (each once) and for the bytes loaded (tests/cpu_emu/run_ycbcr_enc_cases.py); then the same under AddressSanitizer; the
libjpeg-turbo fixture through the kernel; the access widths; and plans corrupted on purpose, which the checks must reject.  The kernel
is also run on the GPU (tests/test_ycbcr_enc_gpu.py)."""
import numpy as np
import pytest

from tests import cpu_emu
from tests import ycbcr_enc_oracle as eo
from tests.cpu_emu import run_ycbcr_enc_cases as rye
from tests.test_ycbcr_enc_oracle import CASES, MATTE, golden_case


@pytest.fixture(scope="module")
def emu_so(tmp_path_factory):
    return cpu_emu.build(str(tmp_path_factory.mktemp("ycbcr_enc_emu")), *rye.SOURCES)


def test_emulated_bgra_to_ycbcr_kernel_matches_the_oracle(emu_so):
    assert rye.run(emu_so, 200) >= 1000


def test_the_libjpeg_turbo_fixture_through_the_emulated_kernel(emu_so):
    """every golden case in one call, the source and each plane at its own phase inside a bitmap of sentinel bytes"""
    L = rye.load(emu_so)
    rng = np.random.default_rng(5)
    jobs = []
    for i, name in enumerate(CASES):
        s, src, y, cb, cr, matte = golden_case(name)
        d, rows, reads, writes = rye.make_job(rng, s, sphase=4 * (i % 4), phases=[i % 16, (i + 5) % 16, (i + 9) % 16],
                                              matte=MATTE if matte else None, src=src)
        for r, p in zip(rows[1:], (y, cb, cr)):                 # the fixture's planes, not the oracle's
            r.view(r.exp)[..., 0] = p
        jobs.append((d, rows, reads, writes))
    ctas, ld, st, n_items, err = rye.launch(L, jobs)
    assert not err and n_items == len(CASES)
    rye.check(jobs, ctas, ld, st)


@pytest.mark.parametrize("sampling", eo.SAMPLINGS)
def test_aligned_rows_take_wide_accesses(emu_so, sampling):
    """At 16-byte source phases and 8-byte plane phases a row's whole runs load 16 bytes at a time and store each plane's bytes in
    one access; only the ragged end of a row (301 = 37 runs + 5 columns) takes word loads and narrower stores."""
    h = 4
    loads, stores = rye.access_widths(emu_so, sampling, w=301, h=h)
    assert loads.get(16, 0) == 2 * 37 * h and loads.get(4, 0) == 5 * h and set(loads) <= {4, 16}, loads
    assert stores.get(8, 0) >= 37 * h and stores.get(1, 0) <= 16 * h, stores


@pytest.mark.parametrize("sampling", eo.SAMPLINGS)
def test_misaligned_rows_are_read_once_in_words(emu_so, sampling):
    """at a source phase no 16-byte load fits, every pixel is one word load: each source byte is read once"""
    loads, _ = rye.access_widths(emu_so, sampling, w=301, h=4, sphase=4, phases=(5, 3, 7))
    assert loads == {4: 301 * 4}, loads


@pytest.mark.parametrize("kind", [1, 2, 3, 4], ids=["wrong_first_cta", "rows_cut_short", "wrong_chroma_plane", "matte_dropped"])
def test_a_sabotaged_plan_is_caught(emu_so, kind):
    assert rye.sabotage_caught(emu_so, kind)


def test_emulated_bgra_to_ycbcr_kernel_under_address_sanitizer(tmp_path):
    so = cpu_emu.build(str(tmp_path), *rye.SOURCES, sanitize=True)
    r = cpu_emu.run_under_asan("run_ycbcr_enc_cases", so, 80)
    assert r.returncode == 0 and "cases bit-exact:" in r.stdout and "AddressSanitizer" not in r.stderr, (r.stdout[-300:], r.stderr[-1500:])
