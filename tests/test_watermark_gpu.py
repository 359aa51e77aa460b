"""Watermarks on the GPU (Batch.watermark -> ifb200_batch_watermark), every case bit for bit against the node-by-node expansion on the
CPU oracle (tests/watermark_oracle.py) AND against the existing route on the device (the Alpha colour chain on a copy of the cropped
watermark, then ifb200_batch_enqueue under the Compose rule): batches of 1, 7, 64 and 1024 frames; mixed frame sizes (several F
groups); Bgr32 and Bgra32 watermarks and frames; opacity none, 0.9, 0.3 and 0; the sRGB working space; a BlendWithMatte frame; cut-out
watermarks; cropped watermark windows at x % 4 = 0..3 in bitmaps with pitches that are not multiples of 16; two watermarks on one frame;
the seven configurations of the reference's visuals/watermark.rs on synthetic frames and logos of their shapes; a bad descriptor,
which changes nothing; and the kernel launches of a call, 1 + 2 x geometries (+1 with an opacity)."""
import ctypes as C

import numpy as np
import pytest

from imageflow_b200 import synth
from tests import watermark_oracle as wo

pytestmark = pytest.mark.gpu


def _ifb():
    import imageflow_b200 as ifb
    return ifb


class Bmp:
    """a host bitmap (h, pitch_px, 4) and the window of it that is used"""
    def __init__(self, arr, am, x0=0, w=None, compose=0, matte=(0, 0, 0, 0)):
        self.arr, self.am, self.x0, self.compose, self.matte = arr, am, x0, compose, tuple(matte)
        self.w = arr.shape[1] - x0 if w is None else w

    @property
    def h(self):
        return self.arr.shape[0]

    def view(self, a):
        return a[:, self.x0:self.x0 + self.w]


def _win(ifb, bm, t):
    return ifb.BitmapWindow(t.data_ptr() + bm.x0 * 4, bm.w, bm.h, t.stride(0), bool(bm.am), ifb.BitmapCompositing(bm.compose),
                            bm.matte, _keep=t)


def _expected(jobs):
    """the node-by-node expansion on the oracle: {id(frame): pixels}"""
    ifb = _ifb()
    out, compose = {}, {}
    for fr, wm, spec in jobs:
        a = out.setdefault(id(fr), fr.arr.copy())
        c = compose.setdefault(id(fr), fr.compose)
        draw = ifb.watermark_layout(fr.w, fr.h, wm.w, wm.h, spec)
        if draw is None:
            continue
        wo.expansion(fr.view(a), c, fr.matte, np.ascontiguousarray(wm.view(wm.arr)), wm.am, draw)
        compose[id(fr)] = wo.BLEND_WITH_SELF
    return out


def _existing_route(b, jobs):
    """the expansion on the device with the existing calls: a copy of the cropped window, the Alpha chain on it, one enqueue"""
    import torch
    ifb = _ifb()
    dev, compose = {}, {}
    for fr, wm, spec in jobs:
        t = dev.setdefault(id(fr), torch.from_numpy(fr.arr.copy()).cuda())
        c = compose.setdefault(id(fr), fr.compose)
        draw = ifb.watermark_layout(fr.w, fr.h, wm.w, wm.h, spec)
        if draw is None:
            continue
        src = torch.from_numpy(np.ascontiguousarray(wm.view(wm.arr))).cuda()
        if draw.crop is not None:
            x1, y1, x2, y2 = draw.crop
            src = src[y1:y2, x1:x2].contiguous()
        sw = ifb.BitmapWindow.from_torch(src, alpha_meaningful=bool(wm.am))
        if draw.opacity is not None:
            b.color_chain([(sw, ifb.ColorFilterSrgb.alpha(draw.opacity))], stream="own")
        cw = _win(ifb, fr, t)
        cw.compose = ifb.BitmapCompositing(wo.drawn_compose(c))
        b.scale_and_render_many([(sw, cw, ifb.ScaleAndRenderParams(x=draw.x, y=draw.y, w=draw.w, h=draw.h, interpolation_filter=draw.filter))],
                                stream="own")
        b.sync()
        compose[id(fr)] = wo.BLEND_WITH_SELF
    return {k: v.cpu().numpy() for k, v in dev.items()}


def _run(jobs, check_launches=None):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    dev = {}
    for fr, wm, _ in jobs:
        for bm in (fr, wm):
            dev.setdefault(id(bm), torch.from_numpy(bm.arr.copy()).cuda())
    wins = {}
    pj = []
    for fr, wm, spec in jobs:
        fw = wins.setdefault(id(fr), _win(ifb, fr, dev[id(fr)]))
        pj.append((fw, _win(ifb, wm, dev[id(wm)]), spec))
    l0 = b.kernel_launches
    out = b.watermark(pj, stream="own")
    b.sync()
    if check_launches is not None:
        assert b.kernel_launches - l0 == check_launches
    exp = _expected(jobs)
    ref = _existing_route(ifb.Batch(0), jobs)
    for fr, wm, spec in jobs:
        got = dev[id(fr)].cpu().numpy()
        assert np.array_equal(got, exp[id(fr)]), ("oracle", fr.w, fr.h, np.argwhere(got != exp[id(fr)])[:3].tolist())
        assert np.array_equal(got, ref[id(fr)]), "existing route"
        assert np.array_equal(dev[id(wm)].cpu().numpy(), wm.arr), "the watermark was written"
    for w, (_, wm, spec) in zip(out, jobs):
        if ifb.watermark_layout(w.w, w.h, wm.w, wm.h, spec) is not None:
            assert w.compose == ifb.BitmapCompositing.BlendWithSelf
    return b, out


def _spec(**kw):
    ifb = _ifb()
    d = dict(fit_box=ifb.WatermarkConstraintBox.image_percentage(0, 0, 90, 90), fit_mode=ifb.WatermarkConstraintMode.Within,
             gravity=ifb.ConstraintGravity.percentage(100, 100), opacity=0.9)
    d.update(kw)
    return ifb.Watermark(**d)


@pytest.mark.parametrize("n", [1, 7, 64, 1024])
def test_batches_one_watermark_many_frames(n):
    logo = Bmp(synth.cutout_np(40, 10, 1), True)
    frames = [Bmp(synth.noise_np(51, 51, 100 + i % 16), i % 2 == 0) for i in range(n)]
    _run([(f, logo, _spec()) for f in frames], check_launches=1 + 2 + 1)


@pytest.mark.parametrize("opacity", [None, 0.9, 0.3, 0.0])
@pytest.mark.parametrize("wm_am", [True, False])
def test_mixed_frame_sizes_formats_and_opacities(opacity, wm_am):
    logo = Bmp(synth.noise_np(64, 30, 5, alpha_mode="mixed"), wm_am)
    frames = [Bmp(synth.cutout_canvas_np(w, h, i), i % 2 == 1) for i, (w, h) in enumerate([(200, 120), (90, 160), (200, 120), (333, 77), (90, 160)])]
    spec = _spec(opacity=opacity, fit_mode=_ifb().WatermarkConstraintMode.Fit)
    _run([(f, logo, spec) for f in frames], check_launches=1 + 2 * 3 + (opacity is not None))


def test_blend_with_matte_frame_and_replace_self_frames():
    logo = Bmp(synth.cutout_np(30, 30, 2), True)
    frames = [Bmp(synth.cutout_canvas_np(70, 50, 1), True, compose=2, matte=(20, 40, 240, 160)),
              Bmp(synth.cutout_canvas_np(70, 50, 2), True, compose=1), Bmp(synth.noise_np(70, 50, 3), False, compose=0)]
    _run([(f, logo, _spec(opacity=0.5)) for f in frames])


@pytest.mark.parametrize("x0", [0, 1, 2, 3])
def test_cropped_windows_at_every_phase_with_unaligned_pitches(x0):
    ifb = _ifb()
    logo = Bmp(synth.cutout_np(103, 41, 9), True, x0=x0, w=97)            # pitch 412 bytes
    frames = [Bmp(synth.cutout_canvas_np(77, 59, s), True) for s in range(3)]   # pitch 308 bytes
    spec = _spec(fit_mode=ifb.WatermarkConstraintMode.FitCrop, fit_box=ifb.WatermarkConstraintBox.image_margins(3, 4, 5, 6),
                 gravity=ifb.ConstraintGravity.percentage(20, 70), opacity=0.3)
    assert ifb.watermark_layout(77, 59, 97, 41, spec).crop is not None
    _run([(f, logo, spec) for f in frames])


def test_two_watermarks_on_one_frame():
    ifb = _ifb()
    a, bb = Bmp(synth.cutout_np(50, 20, 4), True), Bmp(synth.noise_np(33, 33, 6), False)
    frames = [Bmp(synth.noise_np(160, 90, 7), False), Bmp(synth.cutout_canvas_np(160, 90, 8), True)]
    s2 = _spec(fit_box=ifb.WatermarkConstraintBox.canvas_margins(10, 10, 60, 40), gravity=None, opacity=None)
    _run([(frames[0], a, _spec()), (frames[0], bb, s2), (frames[1], a, _spec()), (frames[1], bb, s2), (frames[0], a, s2)])


def test_the_reference_visual_configurations():
    """visuals/watermark.rs: FitCrop into ImagePercentage(30, 50, 90, 90), gravity (100, 100), opacity 0.9, hints sharpen 15 (ignored)
    three times (an 800 x 533 frame, a dice-like 160 x 160 logo); Within into ImagePercentage(0, 0, 90, 90) with opacity 0.9; Within
    into ImageMargins(700, 700, 0, 0); Within with no opacity on a transparent 500 x 600 frame; Within with 0.3 of a Bgr32 logo."""
    ifb = _ifb()
    M, B, G = ifb.WatermarkConstraintMode, ifb.WatermarkConstraintBox, ifb.ConstraintGravity
    dice, small, jpeg = Bmp(synth.cutout_np(160, 160, 11), True), Bmp(synth.cutout_np(60, 45, 12), True), Bmp(synth.noise_np(96, 64, 13), False)
    photo = lambda s: Bmp(synth.noise_np(800, 533, s), False)
    shirt = lambda s: Bmp(synth.cutout_canvas_np(500, 600, s), True)
    hints = object()
    fit = _spec(fit_box=B.image_percentage(30, 50, 90, 90), fit_mode=M.FitCrop, gravity=G.percentage(100, 100), opacity=0.9, hints=hints)
    jobs = [(photo(1), dice, fit), (photo(2), dice, fit), (photo(3), dice, fit),
            (photo(4), small, _spec(hints=hints)),
            (photo(5), small, _spec(fit_box=B.image_margins(700, 700, 0, 0), opacity=0.9)),
            (shirt(6), small, _spec(opacity=None, hints=hints)),
            (shirt(7), jpeg, _spec(opacity=0.3, hints=hints))]
    _run(jobs)


def test_srgb_working_space_through_the_descriptor():
    import torch
    ifb = _ifb()
    from imageflow_b200._lib import WatermarkDesc
    logo, frame = synth.cutout_np(37, 23, 3), synth.cutout_canvas_np(64, 48, 4)
    tl, tf = torch.from_numpy(logo).cuda(), torch.from_numpy(frame).cuda()
    b = ifb.Batch(0)
    for op, linear in ((0.6, 0), (2.0, 0), (float("nan"), 1)):
        tf.copy_(torch.from_numpy(frame))
        d = WatermarkDesc()
        ifb.graphics._fill_desc(d.draw, ifb.BitmapWindow.from_torch(tl, alpha_meaningful=True), ifb.BitmapWindow.from_torch(tf),
                                ifb.ScaleAndRenderParams(x=5, y=6, w=50, h=30, interpolation_filter=ifb.Filter.Ginseng,
                                                         scale_in_colorspace=ifb.WorkingFloatspace(linear)))
        d.opacity = op
        buf = C.create_string_buffer(256)
        assert ifb.lib().ifb200_batch_watermark(b._h, C.byref(d), 1, b.STREAM_OWN, buf, 256) == 0, buf.value
        b.sync()
        exp = frame.copy()
        src = logo.copy()
        if op < 1:
            src, _ = wo.source_of(logo, True, ifb.WatermarkDraw(None, 0, 0, 0, 0, ifb.Filter.Ginseng, op))
        import oracle
        oracle.scale_and_render(src, exp, x=5, y=6, w=50, h=30, filter=4, linear=bool(linear), alpha_meaningful=True, compose=1)
        assert np.array_equal(tf.cpu().numpy(), exp), (op, linear)


def test_a_bad_descriptor_changes_nothing():
    import torch
    ifb = _ifb()
    logo = torch.from_numpy(synth.cutout_np(20, 20, 1)).cuda()
    frames = [torch.from_numpy(synth.noise_np(40, 40, s)).cuda() for s in range(3)]
    before = [f.clone() for f in frames]
    b = ifb.Batch(0)
    spec = _spec()
    jobs = [(ifb.BitmapWindow.from_torch(f), ifb.BitmapWindow.from_torch(logo, alpha_meaningful=True), spec) for f in frames]
    from imageflow_b200._lib import WatermarkDesc
    arr = (WatermarkDesc * 3)()
    for d, (fw, lw, sp) in zip(arr, jobs):
        lay = ifb.watermark_layout(fw.w, fw.h, lw.w, lw.h, sp)
        ifb.graphics._fill_desc(d.draw, lw, fw, ifb.ScaleAndRenderParams(x=lay.x, y=lay.y, w=lay.w, h=lay.h, interpolation_filter=lay.filter))
        d.opacity = 0.5
    arr[2].draw.x = 39                                            # out of bounds
    l0 = b.kernel_launches
    buf = C.create_string_buffer(256)
    rc = ifb.lib().ifb200_batch_watermark(b._h, arr, 3, b.STREAM_OWN, buf, 256)
    b.sync()
    assert rc == 1 and b"out of bounds" in buf.value and b.kernel_launches == l0
    for f, g in zip(frames, before):
        assert torch.equal(f, g)


def test_distinct_watermarks_beyond_the_scratch_bound_run_in_chunks():
    """nine 4K frames of different heights, each with a 1920x1080 watermark fitted to the whole canvas: nine F of about 132 MB, more
    than the 1 GiB a call holds at a time, so the groups run as two chunks (2 x 9 resample launches + 2 composites), bit-exact against
    one batch_enqueue of the same draws"""
    import torch
    ifb = _ifb()
    wm = synth.cutout_torch(1920, 1080, 5)
    ww = ifb.BitmapWindow.from_torch(wm, alpha_meaningful=True)
    spec = ifb.Watermark(fit_box=ifb.WatermarkConstraintBox.canvas_percentage(0, 0, 100, 100), fit_mode=ifb.WatermarkConstraintMode.Fit)
    frames = [synth.noise_torch(3840, 2160 - k, 20 + k) for k in range(9)]
    ref = [f.clone() for f in frames]
    b = ifb.Batch(0)
    wins = [ifb.BitmapWindow.from_torch(f) for f in frames]
    assert sum(ifb.watermark_layout(w.w, w.h, 1920, 1080, spec).w * ifb.watermark_layout(w.w, w.h, 1920, 1080, spec).h * 16
               for w in wins) > 1 << 30
    b.watermark([(w, ww, spec) for w in wins], stream="own")
    b.sync()
    assert b.kernel_launches == 2 * 9 + 2
    jobs = []
    for r in ref:
        d = ifb.watermark_layout(r.shape[1], r.shape[0], 1920, 1080, spec)
        rw = ifb.BitmapWindow.from_torch(r, compose=ifb.BitmapCompositing.BlendWithSelf)
        jobs.append((ww, rw, ifb.ScaleAndRenderParams(x=d.x, y=d.y, w=d.w, h=d.h, interpolation_filter=d.filter)))
    b2 = ifb.Batch(0)
    b2.scale_and_render_many(jobs, stream="own")
    b2.sync()
    for f, r in zip(frames, ref):
        assert torch.equal(f, r)
