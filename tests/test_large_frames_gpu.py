"""Every kernel across its launch seams: frames taller or wider than one grid (65 535 blocks in y), and frames near 2^32 pixels.

Each case is a frame shaped to cross one seam, compared with a plain reference -- the oracle's scale_and_render for the resample
paths, numpy for the exact operations, the committed reference vectors for the block scalers, the oracle for whitespace and colour
-- and each asserts which path ran and how many launches it took, so that no case can pass by taking another route.  Thin frames
cross the seams cheaply: 1 x 2 200 000 is 8.8 MB.  Every window sits inside a larger buffer of sentinel bytes that must come back
unchanged.

The two band tests run color_matrix_kernel and apply_matte_kernel over 65 536 x 65 535 pixels (16 GiB), where a 32-bit grid-stride
index wraps past 2^32 and revisits pixels (tests/test_large_frames_plan.py models it); they skip unless about 20 GiB of device
memory is free, and allocate nothing else of that size."""
import ctypes as C

import numpy as np
import pytest

import oracle
from tests import color_oracle as clo
from tests import orient_oracle as oo
from tests import pixel_convert_oracle as pco
from tests import round_corners_oracle as rco
from tests.test_idct_block_scalers import GOLD

pytestmark = pytest.mark.gpu

MATTE = (40, 120, 250, 200)
SENT = 0xA5                      # sentinel byte around every window
LONG = 2_200_000                 # crosses transpose_locked's 65 535 x 32 = 2 097 120-row launch seam


def _ifb():
    import imageflow_b200 as ifb
    return ifb


def _noise(w, h, seed, alpha="mixed"):
    return oracle.synth_noise(w, h, seed, alpha)


def _dev(a, am=True, pad=3):
    """a device copy of the (h, w, 4) frame `a` at column 1 of a (h, w + pad, 4) tensor of sentinel bytes -> (tensor, window)"""
    import torch
    h, w = a.shape[:2]
    t = torch.full((h, w + pad, 4), SENT, dtype=torch.uint8, device="cuda")
    t[:, 1:1 + w] = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t, _ifb().BitmapWindow.from_torch(t[:, 1:1 + w], alpha_meaningful=am)


def _back(t, w):
    """-> the window's pixels, after checking that every byte around them is still a sentinel"""
    full = t.cpu().numpy()
    assert (full[:, 0] == SENT).all() and (full[:, 1 + w:] == SENT).all(), "a byte outside the window changed"
    return full[:, 1:1 + w]


class _Counts:
    """the Batch counters across a block of calls"""
    NAMES = ("kernel_launches", "fused_jobs", "generic_jobs", "tile_jobs")

    def __init__(self, b):
        self.b = b
        self.at = self._now()

    def _now(self):
        return {n: getattr(self.b, n) for n in self.NAMES}

    def delta(self):
        now = self._now()
        return {n: now[n] - self.at[n] for n in self.NAMES}


def _same(got, want, what):
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.argwhere(np.any(np.asarray(got) != np.asarray(want), axis=-1) if got.ndim == 3 else np.asarray(got) != np.asarray(want))
    assert len(bad) == 0, (what, len(bad), bad[:4].tolist())


# ---------------------------------------------------------------------------------------------------------------- resample
def _resample(b, inp, ow, oh, *, compose=0, canvas=None, flag=None, linear=True):
    """one job through Batch.scale_and_render_many (or _oriented, with `flag`) -> (device result, oracle result, counter deltas)"""
    import torch
    ifb = _ifb()
    cv = np.zeros((oh, ow, 4), np.uint8) if canvas is None else canvas
    src = ifb.BitmapWindow.from_torch(torch.from_numpy(inp).cuda(), alpha_meaningful=True)
    tc = torch.from_numpy(cv.copy()).cuda()
    out = ifb.BitmapWindow.from_torch(tc, compose=ifb.BitmapCompositing(compose), matte_bgra=MATTE)
    p = ifb.ScaleAndRenderParams(w=ow, h=oh, interpolation_filter=ifb.Filter(2),
                                 scale_in_colorspace=ifb.WorkingFloatspace.LinearRGB if linear else ifb.WorkingFloatspace.StandardRGB)
    c = _Counts(b)
    if flag is None:
        b.scale_and_render_many([(src, out, p)], stream="own")
    else:
        b.scale_and_render_oriented([(src, out, p, flag)], stream="own")
    b.sync()
    d = c.delta()
    want = cv.copy()
    oracle.scale_and_render(inp if flag is None else np.ascontiguousarray(oo.gather(inp, flag)), want, w=ow, h=oh, filter=2,
                            alpha_meaningful=True, linear=linear, compose=compose, matte=MATTE)
    got = tc.cpu().numpy()
    del src, out, tc
    torch.cuda.empty_cache()
    return got, want, d


@pytest.mark.parametrize("min_items,compose", [(0, 0), (1 << 20, 1)], ids=["default-bands", "one-band-per-8-rows"])
def test_ring_kernel_on_a_tall_frame(min_items, compose):
    """64 x 140 000 -> 16 x 70 000: in_h and out_h past 65 535 (TMA box rows, vw / vdone of in_h + 32 rows); with OPT_MIN_ITEMS the
    launch takes out_h / 8 = 8 750 bands, so band edges fall every 8 output rows"""
    ifb = _ifb()
    b = ifb.Batch(0)
    assert b.ring_status()[0], b.ring_status()
    b.set_option(ifb.Batch.OPT_MIN_ITEMS, min_items)
    inp = _noise(64, 140_000, 31)
    cv = _noise(16, 70_000, 32) if compose else None
    bands0 = b.host_profile()["ring_bands"]
    got, want, d = _resample(b, inp, 16, 70_000, compose=compose, canvas=cv)
    bands = b.host_profile()["ring_bands"] - bands0
    assert d == {"kernel_launches": 1, "fused_jobs": 1, "generic_jobs": 0, "tile_jobs": 0}, d
    # the band count hv_pick_bands caps at out_h / 8; without OPT_MIN_ITEMS, about one item per device warp
    assert (bands == 8_750) if min_items else (1 <= bands < 8_750), bands
    _same(got, want, ("ring", min_items))
    b.close()


@pytest.mark.parametrize("iw,ih,ow,oh", [(32, 140_000, 16, 20_000), (8, 40_000, 8, 80_000)], ids=["in_h-past-grid", "out_h-past-grid"])
def test_generic_pair_on_a_tall_frame(iw, ih, ow, oh):
    """hpass_generic_kernel's grid.y = min(in_h, 65535) and vpass_generic_kernel's grid.y = min(out_h, 65535), each looping over the rest"""
    ifb = _ifb()
    b = ifb.Batch(0)
    b.set_option(ifb.Batch.OPT_FORCE_GENERIC, 1)
    for linear in (True, False):
        got, want, d = _resample(b, _noise(iw, ih, 33), ow, oh, linear=linear)
        assert d == {"kernel_launches": 2, "fused_jobs": 0, "generic_jobs": 1, "tile_jobs": 0}, d
        _same(got, want, ("generic", iw, ih, ow, oh, linear))
    b.close()


@pytest.mark.parametrize("iw,ih,ow,oh", [(16, 40_000, 32, 80_000), (40_000, 2, 80_000, 4)], ids=["tiles_y-past-grid", "tiles_x-past-grid"])
def test_tile_kernel_up_scales_past_the_resident_grid(iw, ih, ow, oh):
    """2 500 tile rows of one tile column (step_x == 0), and 1 250 tile columns of one tile row (step_y == 0): both far more tiles
    than the resident CTAs, which walk them"""
    ifb = _ifb()
    b = ifb.Batch(0)
    got, want, d = _resample(b, _noise(iw, ih, 34), ow, oh)
    assert d == {"kernel_launches": 1, "fused_jobs": 0, "generic_jobs": 0, "tile_jobs": 1}, d
    _same(got, want, ("tile", iw, ih, ow, oh))
    b.close()


@pytest.mark.parametrize("flag", [5, 6, 7, 8])
def test_oriented_generic_pair_with_out_w_past_the_grid(flag):
    """flags 5..8 (a transposed source read): the H pass runs one output column per blockIdx.y, grid.y = min(out_w, 65535); the
    stored 4 x 40 000 frame is 40 000 x 4 oriented and up-scaled to 80 000 x 6 (oriented up-scales take the generic pair)"""
    ifb = _ifb()
    b = ifb.Batch(0)
    got, want, d = _resample(b, _noise(4, 40_000, 35 + flag), 80_000, 6, flag=flag)
    assert d == {"kernel_launches": 2, "fused_jobs": 0, "generic_jobs": 1, "tile_jobs": 0}, d
    _same(got, want, ("oriented", flag))
    b.close()


@pytest.mark.parametrize("opacity,launches", [(None, 3), (0.5, 4)], ids=["opaque", "opacity"])
def test_watermark_resample_of_a_tall_box(opacity, launches):
    """a 4 x 70 000 watermark drawn over the whole of an 8 x 140 000 frame: the watermark's generic H pass runs grid.y = min(in_h,
    65535) over 70 000 rows and vpass_f_kernel grid.y = min(out_h, 65535) over 140 000 rows, then one composite launch (and one
    colour-chain launch before them for the opacity); against the node-by-node expansion on the oracle"""
    import torch
    from tests import watermark_oracle as wo
    ifb = _ifb()
    b = ifb.Batch(0)
    frame, wm = _noise(8, 140_000, 55), _noise(4, 70_000, 56)
    spec = ifb.Watermark(fit_box=ifb.WatermarkConstraintBox.canvas_percentage(0, 0, 100, 100),
                         fit_mode=ifb.WatermarkConstraintMode.Distort, opacity=opacity)
    draw = ifb.watermark_layout(8, 140_000, 4, 70_000, spec)
    assert (draw.w, draw.h) == (8, 140_000), draw
    tf, wf = _dev(frame)
    tw, ww = _dev(wm)
    c = _Counts(b)
    b.watermark([(wf, ww, spec)], stream="own")
    b.sync()
    assert c.delta()["kernel_launches"] == launches
    want = frame.copy()
    wo.expansion(want, wo.REPLACE_SELF, (0, 0, 0, 0), wm, True, draw)
    _same(_back(tf, 8), want, ("watermark", opacity))
    _same(_back(tw, 4), wm, "the watermark changed")
    del tf, tw
    torch.cuda.empty_cache()
    b.close()


# ---------------------------------------------------------------------------------------------------------------- exact operations
@pytest.mark.parametrize("w,h,launches", [(1, LONG, 2), (LONG, 1, 1)], ids=["one-long-column", "one-long-row"])
def test_transpose_of_a_long_row_and_column(w, h, launches):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    a = _noise(w, h, 41)
    ts, src = _dev(a)
    td, dst = _dev(np.zeros((w, h, 4), np.uint8))
    td[:, 1:1 + h].fill_(SENT)                      # the destination is all sentinel until the kernel writes it
    c = _Counts(b)
    b.transpose(src, dst, stream="own")
    b.sync()
    assert c.delta()["kernel_launches"] == launches
    _same(_back(td, h), a.transpose(1, 0, 2), ("transpose", w, h))
    _same(_back(ts, w), a, "the source changed")
    del ts, td
    torch.cuda.empty_cache()
    b.close()


@pytest.mark.parametrize("w,h", [(1, LONG), (LONG, 1), (3, 700_001)], ids=["one-long-column", "one-long-row", "three-columns"])
def test_flips_of_a_long_row_and_column(w, h):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    a = _noise(w, h, 42)
    for vertical in (False, True):
        t, win = _dev(a)
        c = _Counts(b)
        (b.flip_vertical if vertical else b.flip_horizontal)(win, stream="own")
        b.sync()
        moves = (h // 2 if vertical else w // 2) > 0
        assert c.delta()["kernel_launches"] == (1 if moves else 0), (vertical, w, h)
        _same(_back(t, w), a[::-1] if vertical else a[:, ::-1], ("flip", vertical, w, h))
        del t
    torch.cuda.empty_cache()
    b.close()


@pytest.mark.parametrize("w,h", [(1, 1_000_003), (1_000_003, 1)], ids=["one-long-column", "one-long-row"])
def test_orient_every_flag_in_one_launch(w, h):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    a = _noise(w, h, 43)
    ts, src = _dev(a)
    outs = []
    for flag in range(1, 9):
        ow, oh = (h, w) if flag >= 5 else (w, h)
        outs.append(_dev(np.full((oh, ow, 4), SENT, np.uint8)) + (ow, flag))
    c = _Counts(b)
    b.orient([(src, o[1], o[3]) for o in outs], stream="own")
    b.sync()
    assert c.delta()["kernel_launches"] == 1
    for t, _, ow, flag in outs:
        _same(_back(t, ow), oo.gather(a, flag), ("orient", flag, w, h))
    _same(_back(ts, w), a, "the source changed")
    del ts, outs
    torch.cuda.empty_cache()
    b.close()


@pytest.mark.parametrize("w,h", [(1, 1_000_003), (1_000_003, 1)], ids=["one-long-column", "one-long-row"])
def test_canvas_fill_copy_expand_in_one_launch(w, h):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    a, bg = _noise(w, h, 44), _noise(w, h, 45)
    color = (9, 8, 7, 255)
    # FillRect inside the window, leaving a margin of its long side
    tf, wf = _dev(bg)
    x1, y1, x2, y2 = (0, 5, 1, h - 3) if w == 1 else (5, 0, w - 3, 1)
    want_fill = bg.copy(); want_fill[y1:y2, x1:x2] = color
    # CopyRectToCanvas of the whole frame to (2, 3) of a larger canvas
    tcv, wcv = _dev(_noise(w + 4, h + 5, 46))
    want_copy = tcv[:, 1:1 + w + 4].cpu().numpy().copy(); want_copy[3:3 + h, 2:2 + w] = a
    ti, wi = _dev(a)
    # ExpandCanvas by (1, 2, 3, 4) into a given canvas
    te, we = _dev(np.zeros((h + 6, w + 4, 4), np.uint8))
    want_exp = np.empty((h + 6, w + 4, 4), np.uint8); want_exp[...] = color; want_exp[2:2 + h, 1:1 + w] = a
    c = _Counts(b)
    b.canvas([ifb.FillRect(wf, x1, y1, x2, y2, color), ifb.CopyRectToCanvas(wi, wcv, 0, 0, w, h, 2, 3),
              ifb.ExpandCanvas(wi, 1, 2, 3, 4, color, canvas=we)], stream="own")
    b.sync()
    assert c.delta()["kernel_launches"] == 1
    _same(_back(tf, w), want_fill, "fill")
    _same(_back(tcv, w + 4), want_copy, "copy")
    _same(_back(te, w + 4), want_exp, "expand")
    _same(_back(ti, w), a, "the source changed")
    del tf, tcv, ti, te
    torch.cuda.empty_cache()
    b.close()


@pytest.mark.parametrize("w,h", [(1, 1_000_003), (1_000_003, 1)], ids=["one-long-column", "one-long-row"])
def test_pixel_convert_every_op_in_one_launch(w, h):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    rng = np.random.default_rng(47)
    jobs, checks = [], []
    for op in pco.OPS:
        cs, cd = pco.CHANNELS[op]
        for opaque in (False, True):
            src = rng.integers(0, 256, (h, w, cs), dtype=np.uint8)
            ts = torch.from_numpy(src).cuda()
            td = torch.full((h, w + 1, cd), SENT, dtype=torch.uint8, device="cuda")
            jobs.append(ifb.graphics._PIXEL_OPS[op](ts, td[:, :w], opaque))
            checks.append((op, opaque, src, ts, td))
    c = _Counts(b)
    b.pixel_convert(jobs, stream="own")
    b.sync()
    assert c.delta()["kernel_launches"] == 1
    for op, opaque, src, ts, td in checks:
        full = td.cpu().numpy()
        assert (full[:, w:] == SENT).all(), ("a byte outside the rows changed", op)
        _same(full[:, :w], pco.convert(op, src, opaque), ("pixel_convert", op, opaque))
        assert np.array_equal(ts.cpu().numpy(), src), ("the source changed", op)
    del jobs, checks
    torch.cuda.empty_cache()
    b.close()


@pytest.mark.parametrize("w,h", [(1, 1_000_003), (1_000_003, 1), (5, 400_001)], ids=["one-long-column", "one-long-row", "five-columns"])
def test_round_corners_in_one_launch(w, h):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    cases = [(ifb.RoundCornersMode.pixels(3.0), (10, 20, 30, 255)), (ifb.RoundCornersMode.circle(), (0, 0, 0, 0)),
             (ifb.RoundCornersMode.pixels_custom(2.0, 0.0, 7.5, 1.0), (200, 100, 50, 128))]
    frames = []
    for i, (mode, matte) in enumerate(cases):
        a = _noise(w, h, 48 + i)
        want = a.copy()
        rco.round_corners(want, mode.kind, mode.radius, matte)
        t, win = _dev(a)
        frames.append((t, win, mode, matte, want))
    writes = any(not np.array_equal(want, _noise(w, h, 48 + i)) for i, (*_, want) in enumerate(frames))
    c = _Counts(b)
    b.round_corners([(win, mode, matte) for _, win, mode, matte, _ in frames], stream="own")
    b.sync()
    assert c.delta()["kernel_launches"] == (1 if writes else 0)
    for t, _, mode, matte, want in frames:
        _same(_back(t, w), want, ("round_corners", mode, matte))
    del frames
    torch.cuda.empty_cache()
    b.close()


def test_block_scalers_past_65535_block_rows():
    """65 544 block rows (two launches): the committed plane's first four block columns repeated down the column, so every output
    block must equal the reference's output for its block in tests/golden/idct_golden.npz"""
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    reps = 65_544 // 8                              # the plane has 8 block rows
    plane = np.ascontiguousarray(GOLD["plane"][:, :32])
    tall = np.tile(plane, (reps, 1))
    tin = torch.from_numpy(tall).cuda()
    for s in (0, 1):
        for n in range(1, 8):
            pitch = 4 * n + 3                        # padded rows of sentinel bytes
            tout = torch.full((65_544 * n, pitch), SENT, dtype=torch.uint8, device="cuda")
            c = _Counts(b)
            b.block_scale(tin.data_ptr(), 32, 4, 65_544, tout.data_ptr(), pitch, n, bool(s), stream="own")
            b.sync()
            assert c.delta()["kernel_launches"] == 2
            got = tout.cpu().numpy()
            assert (got[:, 4 * n:] == SENT).all(), (s, n)
            want = np.tile(GOLD[f"out_{s}_{n}"][:, :4 * n], (reps, 1))
            bad = np.argwhere(got[:, :4 * n] != want)
            assert len(bad) == 0, (s, n, len(bad), (bad[:4] // [n, n]).tolist())
            del tout
    del tin
    torch.cuda.empty_cache()
    b.close()


# ---------------------------------------------------------------------------------------------------------------- whitespace
def test_whitespace_past_524280_rows():
    """8 x 600 000 white frame with content on both sides of the codes kernel's 65 535 x 8 = 524 280-row launch seam: codes against
    the oracle's, and detect_content_many's rectangle and visited count against oracle.detect_content"""
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    w, h, seam = 8, 600_000, 65_535 * 8
    rng = np.random.default_rng(51)
    for y0, y1 in ((seam - 40, seam + 40), (seam - 1, seam + 1), (seam + 2, seam + 9), (seam - 9, seam - 2), (1_000, seam + 1)):
        a = np.full((h, w, 4), 255, np.uint8)
        a[y0:y1, 2:6] = rng.integers(0, 200, (y1 - y0, 4, 4), dtype=np.uint8)
        t, win = _dev(a)
        codes = torch.full((h * w,), SENT, dtype=torch.uint8, device="cuda")
        c = _Counts(b)
        b.whitespace_codes(win, codes.data_ptr(), 1, stream="own")
        b.sync()
        assert c.delta()["kernel_launches"] == 2
        got = codes.cpu().numpy().reshape(h, w)
        want = oracle.whitespace_codes(a, 1, True)
        _same(got, want, ("codes", y0, y1))
        rect_want, visited_want = oracle.detect_content(a, 1, True)
        assert ifb.detect_content_from_codes(got) == (rect_want, visited_want), (y0, y1)
        c = _Counts(b)
        rects, visited = b.detect_content_many([(win, 1)], visited=True, stream="own")
        assert c.delta()["kernel_launches"] == 2
        assert (rects[0], visited[0]) == (rect_want, visited_want), (y0, y1, rects, visited, rect_want, visited_want)
        del t, codes
    torch.cuda.empty_cache()
    b.close()


# ---------------------------------------------------------------------------------------------------------------- colour
THIN = [(1, LONG), (LONG, 1), (3, 700_001)]
THIN_IDS = ["one-long-column", "one-long-row", "three-columns"]


@pytest.mark.parametrize("w,h", THIN, ids=THIN_IDS)
def test_color_chain_matrix_and_white_balance(w, h):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    a = _noise(w, h, 52, "opaque")
    steps = [ifb.ColorMatrixSrgb(ifb.color_filter_matrix(9, -0.4)), ifb.WhiteBalanceHistogramAreaThresholdSrgb(None)]
    want, _, _ = clo.run_chain(a, clo.of_product(steps), True)
    t, win = _dev(a)
    c = _Counts(b)
    b.color_chain([(win, steps)], stream="own")
    b.sync()
    assert c.delta()["kernel_launches"] == 3        # histogram, byte maps, the chain
    _same(_back(t, w), want, ("color_chain", w, h))
    del t
    torch.cuda.empty_cache()
    b.close()


@pytest.mark.parametrize("w,h", THIN, ids=THIN_IDS)
def test_color_matrix_and_apply_matte_on_the_device_and_from_the_host(w, h):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    a = _noise(w, h, 53)
    m = ifb.color_filter_matrix(0)
    want_m = a.copy(); oracle.color_matrix(want_m, m)
    want_a = a.copy(); oracle.apply_matte(want_a, MATTE, True)
    t, win = _dev(a)
    c = _Counts(b)
    b.color_matrix(win.ptr, w, h, win.stride, m, stream="own")
    b.sync()
    assert c.delta()["kernel_launches"] == 1
    _same(_back(t, w), want_m, ("color_matrix", w, h))
    t, win = _dev(a)
    err = C.create_string_buffer(512)
    c = _Counts(b)
    rc = ifb.lib().ifb200_batch_apply_matte(b._h, win.ptr, w, h, win.stride, (C.c_uint8 * 4)(*MATTE), 1, b._stream("own"), err, 512)
    assert rc == 0, err.value
    b.sync()
    assert c.delta()["kernel_launches"] == 1
    _same(_back(t, w), want_a, ("apply_matte", w, h))
    del t
    # the host drop-ins (ifb200_color_matrix_bgra8, ifb200_apply_matte_bgra8) on a padded host window
    host = np.full((h, w + 3, 4), SENT, np.uint8)
    host[:, 1:1 + w] = a
    ifb.window_bgra32_apply_color_matrix(ifb.BitmapWindow.from_numpy(host[:, 1:1 + w]), m)
    assert (host[:, 0] == SENT).all() and (host[:, 1 + w:] == SENT).all()
    _same(host[:, 1:1 + w], want_m, ("host color_matrix", w, h))
    host[:, 1:1 + w] = a
    ifb.apply_matte(ifb.BitmapWindow.from_numpy(host[:, 1:1 + w], alpha_meaningful=True), MATTE)
    assert (host[:, 0] == SENT).all() and (host[:, 1 + w:] == SENT).all()
    _same(host[:, 1:1 + w], want_a, ("host apply_matte", w, h))
    torch.cuda.empty_cache()
    b.close()


# ---------------------------------------------------------------------------------------------------------------- the 2^32 - S band
BAND_W, BAND_H = 65_536, 65_535                  # 2^32 - 65 536 pixels: above 2^32 - S for any grid of more than 65 536 threads
BAND_FREE = 20 << 30


def _band_frame(pixel):
    """a BAND_W x BAND_H frame (16 GiB) on cuda:0 whose every pixel holds the BGRA bytes `pixel`, as (H, W) int32 words"""
    import torch
    free, _ = torch.cuda.mem_get_info(0)
    if free < BAND_FREE:
        pytest.skip(f"the {BAND_W} x {BAND_H} band frame takes 16 GiB; {free / 2**30:.1f} GiB of device memory is free, 20 GiB wanted")
    t = torch.empty((BAND_H, BAND_W), dtype=torch.int32, device="cuda:0")
    t.fill_(_word(pixel))
    return t


def _word(pixel):
    return int(np.frombuffer(bytes(pixel), np.int32)[0])


def _band_check(t, once, twice):
    """counts the pixels that are not `once` (and of them, those that are `twice`) in row chunks on the device, then checks sampled
    pixels -- the first rows, which every wrapped thread revisits first, and random ones -- on the host"""
    import torch
    wrong = doubled = 0
    w_once, w_twice = _word(once), _word(twice)
    for y0 in range(0, BAND_H, 2048):
        ch = t[y0:y0 + 2048]
        wrong += int((ch != w_once).sum())
        doubled += int((ch == w_twice).sum())
    rng = np.random.default_rng(61)
    ys = np.concatenate([np.zeros(64, np.int64), np.ones(64, np.int64), rng.integers(0, BAND_H, 256)])
    xs = np.concatenate([np.arange(64), np.arange(64), rng.integers(0, BAND_W, 256)])
    sample = t[torch.from_numpy(ys).cuda(), torch.from_numpy(xs).cuda()].cpu().numpy().view(np.uint8).reshape(-1, 4)
    bad_samples = int(np.any(sample != np.array(once, np.uint8), axis=1).sum())
    print(f"band {BAND_W} x {BAND_H}: {wrong} pixels differ from one application, {doubled} of them equal two applications; "
          f"{bad_samples} of {len(ys)} sampled pixels differ from the oracle")
    assert (wrong, bad_samples) == (0, 0), (wrong, doubled, bad_samples)


def _once_twice(fn, pixel):
    px = np.array([[pixel]], np.uint8)
    fn(px); once = tuple(int(v) for v in px[0, 0])
    fn(px); twice = tuple(int(v) for v in px[0, 0])
    assert once != twice, "the content must not be idempotent under the op"
    return once, twice


def test_color_matrix_in_the_band_below_2_32():
    """a bias of one level on r, g and b: a pixel the kernel reaches twice is one level off"""
    import torch
    ifb = _ifb()
    pixel = (10, 20, 30, 200)
    m = np.eye(5, dtype=np.float32)
    m[4, :3] = np.float32(1.0 / 255.0)
    once, twice = _once_twice(lambda px: oracle.color_matrix(px, m), pixel)
    t = _band_frame(pixel)
    b = ifb.Batch(0)
    try:
        c = _Counts(b)
        b.color_matrix(t.data_ptr(), BAND_W, BAND_H, BAND_W * 4, m, stream="own")
        b.sync()
        assert c.delta()["kernel_launches"] == 1
        _band_check(t, once, twice)
    finally:
        b.close()
        del t
        torch.cuda.empty_cache()


def test_apply_matte_in_the_band_below_2_32():
    """a pixel alpha of 128 over a matte alpha of 200: a pixel the kernel reaches twice has a different alpha (0 and 255 would be
    fixed points)"""
    import torch
    ifb = _ifb()
    pixel, matte = (10, 20, 30, 128), (200, 100, 50, 200)
    once, twice = _once_twice(lambda px: oracle.apply_matte(px, matte, True), pixel)
    t = _band_frame(pixel)
    b = ifb.Batch(0)
    try:
        err = C.create_string_buffer(512)
        c = _Counts(b)
        rc = ifb.lib().ifb200_batch_apply_matte(b._h, t.data_ptr(), BAND_W, BAND_H, BAND_W * 4, (C.c_uint8 * 4)(*matte), 1,
                                                b._stream("own"), err, 512)
        assert rc == 0, err.value
        b.sync()
        assert c.delta()["kernel_launches"] == 1
        _band_check(t, once, twice)
    finally:
        b.close()
        del t
        torch.cuda.empty_cache()
