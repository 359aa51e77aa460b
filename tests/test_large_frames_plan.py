"""The launch seams of frames taller or wider than one grid, on the CPU: (1) the ring kernel's host tables for tall geometries
(ifb200_hv_plan_tables) and (2) plain Python models of the index arithmetic by which the engine cuts work at the grid limits and
its kernels loop over what one grid cannot hold.  Each model enumerates the indices every launch (and every thread of a grid-stride
loop) touches, and asserts that every pixel, row or tile is visited exactly once at and around each seam.

The grid-stride model is the CPU-side evidence for the 32-bit loop counter that color_matrix_kernel and apply_matte_kernel once
had: on a grid of S threads, a frame of more than 2^32 - S pixels makes some thread's `i += S` wrap past 2^32 to an index below
the frame's size, and that thread starts a second pass over pixels that are already done.  tests/test_large_frames_gpu.py runs the
same frames on the device."""
import ctypes as C

import numpy as np
import pytest

from tests import cpu_emu

GRID_Y = 65535                     # the largest gridDim.y (and gridDim.z)
H100_SXM_SMS, H100_PCIE_SMS = 132, 114


# ---------------------------------------------------------------------------------------------- (1) ring kernel tables of tall frames
class _Band(C.Structure):                           # imageflow_b200/csrc/ifb_hv_kernel.cuh HvBandDev
    _fields_ = [(n, C.c_int32) for n in ("Y0", "Y1", "Yf", "vslot0", "j0", "nrows", "pad0", "pad1")]


class _Strip(C.Structure):                          # HvStripDev
    _fields_ = [(n, C.c_int32) for n in ("X0", "X1", "Xf", "hslot0", "k0", "nst", "pad0", "pad1")]


@pytest.mark.parametrize("iw,ih,ow,oh,alpha", [
    (64, 140_000, 16, 70_000, True),                # the GPU test's tall ring case: in_h and out_h past 65 535
    (64, 140_000, 16, 70_000, False),
    (32, 65_536, 8, 65_536 // 3, True),             # in_h just past one grid
    (16, 300_000, 16, 100_000, False),              # a 1:1 width, in_h past 2^18
])
@pytest.mark.parametrize("pairs", [1, 7, 8_750])
def test_ring_plans_of_tall_frames(iw, ih, ow, oh, alpha, pairs):
    import imageflow_b200 as ifb
    pairs = min(pairs, max(1, oh // 8))              # the engine caps the band count at out_h / 8 (hv_pick_bands)
    info, blob = cpu_emu.hv_plan(ifb, iw, ih, ow, oh, 2, n_bands=pairs, alpha=alpha)
    assert info.ok and blob is not None, (iw, ih, ow, oh)
    assert info.av in (4, 6) and info.n_strips >= 1 and info.n_bands == pairs
    strips = (_Strip * info.n_strips).from_buffer_copy(blob[info.o_strips:info.o_strips + info.n_strips * C.sizeof(_Strip)].tobytes())
    assert strips[0].X0 == 0 and strips[-1].X1 == ow
    assert all(a.X1 == b.X0 for a, b in zip(strips[:-1], strips[1:]))
    # vdone: per source row, the output rows whose V window ends there (+ 32 rows of zeros behind the last)
    vdone = blob[info.o_vdone:info.o_vdone + ih + 32]
    assert int(vdone.sum(dtype=np.int64)) == oh and not vdone[ih:].any()
    assert int(np.flatnonzero(vdone)[-1]) < ih
    bands = (_Band * info.n_bands).from_buffer_copy(blob[info.o_bands:info.o_bands + info.n_bands * C.sizeof(_Band)].tobytes())
    rows = [(b.Y0, b.Y1) for b in bands if b.Y1 > b.Y0]
    assert rows[0][0] == 0 and rows[-1][1] == oh and all(a[1] == b[0] for a, b in zip(rows[:-1], rows[1:]))
    for b in bands:
        if b.Y1 > b.Y0:
            assert 0 <= b.j0 and b.j0 + b.nrows <= ih and b.Yf <= b.Y0 and b.vslot0 == b.Yf % info.av
            # the band's source rows hold the V windows of its output rows: the rows vdone says complete in them add up to at least
            # the band's own (rows of the band before it may complete there too)
            assert int(vdone[b.j0:b.j0 + b.nrows].sum(dtype=np.int64)) >= b.Y1 - b.Y0


@pytest.fixture(scope="module")
def hv_emu(tmp_path_factory):
    return cpu_emu.load_hv(cpu_emu.build(str(tmp_path_factory.mktemp("hv_emu")), "hv_kernel_emu.cc"))


@pytest.mark.parametrize("grid,pairs", [(1, 1), (2, 4)])
def test_emulated_ring_kernel_on_a_frame_just_past_one_grid(hv_emu, grid, pairs):
    """the ring kernel's CUDA source run on the CPU (tests/cpu_emu) over 16 x 65 600 -> 8 x 32 800: source rows past 65 535 stream
    through its TMA boxes and V ring; bit-exact against the oracle (about two seconds a case)"""
    import imageflow_b200 as ifb
    import oracle
    inp = oracle.synth_noise(16, 65_600, 57, "mixed")
    cv = np.zeros((32_800, 8, 4), np.uint8)
    outs = cpu_emu.run_hv(hv_emu, ifb, inp, cv, alpha_meaningful=True, grid=grid, n_bands=pairs)
    assert outs is not None, "not a ring-kernel geometry"
    want = cv.copy()
    oracle.scale_and_render(inp, want, filter=2, alpha_meaningful=True)
    bad = np.argwhere(np.any(outs[0] != want, axis=2))
    assert len(bad) == 0, (len(bad), bad[:4].tolist())


# ---------------------------------------------------------------------------------------------- (2) models of the seams
def _stride_passes(total, S, bits):
    """The loop `for (i = t; i < total; i += S)` of each thread t < S of a grid of S threads, with i an unsigned `bits`-bit integer.
    -> every pass as (thread, first index): a thread's first pass starts at t; when the step after its last index wraps past
    2^bits to an index below `total`, the thread starts another pass there."""
    assert bits in (32, 64) and total < 1 << 40
    t = np.arange(min(S, total), dtype=np.int64)
    out_t, out_s = [t], [t.copy()]
    start = t.copy()
    while len(start):
        last = start + (total - 1 - start) // S * S
        nxt = last + S if bits == 64 else (last + S) & 0xFFFFFFFF     # the index the step after the last one holds in `bits` bits
        again = nxt < total
        t, start = t[again], nxt[again]
        out_t.append(t); out_s.append(start.copy())
    return np.concatenate(out_t), np.concatenate(out_s)


def _stride_visits(total, S, bits, lo, hi):
    """-> (visits of each index in [lo, hi), total visits over the whole frame); hi - lo <= S, so one pass touches at most one index"""
    assert hi - lo <= S
    _, s = _stride_passes(total, S, bits)
    n_in_pass = (total - 1 - s) // S + 1
    k = np.maximum(0, -(-(lo - s) // S))              # the first step of each pass at or after lo
    i = s + k * S
    hit = (i < hi) & (i < total)
    counts = np.bincount((i[hit] - lo).astype(np.int64), minlength=hi - lo)
    return counts, int(n_in_pass.sum())


def _grid_threads(total, sms):
    """the threads color_matrix_locked / apply_matte_locked launch: min(ceil(total / 256), 16 * SMs) blocks of 256"""
    return min((total + 255) // 256, 16 * sms) * 256


def _extra_visits(total, sms, bits):
    S = _grid_threads(total, sms)
    _, visits = _stride_visits(total, S, bits, 0, 1)
    return visits - total


@pytest.mark.parametrize("sms", [H100_SXM_SMS, H100_PCIE_SMS])
@pytest.mark.parametrize("w,h", [(65_536, 65_535), (65_535, 65_535), (65_536, 65_528), (1, 2_200_000), (2_200_000, 1)])
def test_a_64_bit_grid_stride_visits_every_pixel_once(sms, w, h):
    """a loop that cannot wrap: the visits of the kernels' counted loop (each thread's (total - 1 - first) / S + 1 steps)"""
    total = w * h
    S = _grid_threads(total, sms)
    assert _extra_visits(total, sms, 64) == 0
    for lo in (0, total - S, max(0, (1 << 32) - S - 1000)):         # the first indices, the last, and the band below 2^32 - S
        lo = max(0, min(lo, total - min(S, 4096)))
        hi = min(total, lo + min(S, 4096))
        counts, _ = _stride_visits(total, S, 64, lo, hi)
        assert (counts == 1).all(), (w, h, lo)


@pytest.mark.parametrize("sms", [H100_SXM_SMS, H100_PCIE_SMS])
def test_a_32_bit_grid_stride_revisits_pixels_only_in_the_band_below_2_32(sms):
    """the loop form color_matrix_kernel / apply_matte_kernel had: exact below 2^32 - S, wrong inside the band (the 16 GiB frames of
    tests/test_large_frames_gpu.py)"""
    S = 16 * sms * 256
    for total in (2_200_000, 7680 * 4320, (1 << 32) - S - 1, (1 << 32) - S):
        assert _extra_visits(total, sms, 32) == 0, total
    for w, h in ((65_536, 65_528), (65_535, 65_535), (65_536, 65_535)):
        total = w * h
        if total <= (1 << 32) - _grid_threads(total, sms):
            continue
        assert _extra_visits(total, sms, 32) > 0, (w, h)
        counts, _ = _stride_visits(total, S, 32, 0, 4096)             # the wrapped threads start again at the first indices
        assert counts.max() > 1, (w, h)
    # the 132-SM counts the kernel's comment and the GPU test report against
    if sms == H100_SXM_SMS:
        assert _extra_visits(65_536 * 65_535, sms, 32) > 7 * 65_536 * 65_535 * 0.9
        assert _extra_visits(65_536 * 65_535, sms, 64) == 0


def _cut_rows(h, rows_per_launch, rows_per_block):
    """the host loops of transpose_locked, block_scale_locked and whitespace_codes_locked: launches of at most rows_per_launch rows,
    each with grid.y = ceil(rows / rows_per_block) blocks of rows_per_block rows.  -> (visits per row, launches, largest grid.y)"""
    visits = np.zeros(h, np.int32)
    launches, gy_max = 0, 0
    for y0 in range(0, h, rows_per_launch):
        rows = min(rows_per_launch, h - y0)
        gy = (rows + rows_per_block - 1) // rows_per_block
        gy_max = max(gy_max, gy)
        r = y0 + np.arange(gy * rows_per_block)                       # every row a block of the launch covers ...
        visits[r[r < y0 + rows]] += 1                                  # ... that the launch's bound lets through
        launches += 1
    return visits, launches, gy_max


@pytest.mark.parametrize("what,rpl,rpb", [("transpose", GRID_Y * 32, 32), ("block_scale (block rows)", GRID_Y, 1),
                                          ("whitespace_codes", GRID_Y * 8, 8)])
def test_launch_cuts_cover_every_row_once(what, rpl, rpb):
    for h in (1, rpb, rpl - 1, rpl, rpl + 1, 2 * rpl + 7, 2_200_000 if rpb == 32 else 600_000):
        visits, launches, gy = _cut_rows(h, rpl, rpb)
        assert (visits == 1).all(), (what, h)
        assert launches == -(-h // rpl) and gy <= GRID_Y, (what, h)
    # the GPU test's frames: 2 200 000 rows (transpose), 65 544 block rows (block scalers), 600 000 rows (whitespace codes)
    h = {32: 2_200_000, 1: 65_544, 8: 600_000}[rpb]
    assert _cut_rows(h, rpl, rpb)[1] == 2


@pytest.mark.parametrize("n", [1, 65_535, 65_536, 70_000, 140_000, 200_001])
def test_grid_y_loops_visit_every_row_once(n):
    """hpass_generic_kernel / hpass_oriented_kernel / vpass_generic_kernel, and the watermark's H pass and vpass_f_kernel:
    grid.y = min(n, 65535), rows blockIdx.y + k * gridDim.y"""
    gy = min(n, GRID_Y)
    visits = np.zeros(n, np.int32)
    for by in range(gy):
        visits[by::gy] += 1
    assert (visits == 1).all()


def _tile_walk(tiles_x, tiles_y, n_jobs, grid):
    """fused_tile2_kernel's walk over (job, tile row, tile column), advanced without dividing (ifb_tile2_kernel.cuh)"""
    seen = np.zeros((n_jobs, tiles_y, tiles_x), np.int32)
    step_y, step_x = grid // tiles_x, grid % tiles_x
    for bx in range(grid):
        ty, tx, ji = bx // tiles_x, bx % tiles_x, 0
        while True:
            if tx >= tiles_x:
                tx -= tiles_x; ty += 1
            while ty >= tiles_y:
                ty -= tiles_y; ji += 1
            if ji >= n_jobs:
                break
            seen[ji, ty, tx] += 1
            tx += step_x; ty += step_y
    return seen


@pytest.mark.parametrize("tiles_x,tiles_y,n_jobs,grid", [
    (1250, 1, 1, 264),           # out_w 80 000: tiles_x beyond the resident grid, step_y == 0
    (1250, 2, 3, 264),
    (1, 2500, 1, 264),           # out_h 80 000: one tile column, step_x == 0
    (7, 400, 2, 264),
    (264, 3, 2, 264),            # tiles_x == grid: step_y == 1, step_x == 0
    (265, 3, 2, 264),            # one more than the grid: step_y == 0, step_x == 264
])
def test_tile_walk_visits_every_tile_once(tiles_x, tiles_y, n_jobs, grid):
    grid = min(grid, tiles_x * tiles_y * n_jobs)                      # the engine launches min(total, resident) CTAs
    seen = _tile_walk(tiles_x, tiles_y, n_jobs, grid)
    assert (seen == 1).all(), np.argwhere(seen != 1)[:4].tolist()
