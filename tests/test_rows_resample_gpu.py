"""The rows resample on the GPU (Batch.scale_and_render_rows -> ifb200_batch_enqueue_rows), bit for bit against both the two-step
route on the device (Batch.pixel_convert into a BGRA scratch frame, then Batch.scale_and_render_many) and the oracle's
scale_and_render of the rows converted in numpy: RGB24 and RGBA32 on the ring kernel's row forms and on the generic pair (the
counters confirm which ran), both channel counts and working spaces, every compositing mode, sharpen, the fused colour matrix,
cut-out alpha, sub-windows at every byte phase, pitches that are not multiples of 16, an up-scale, 1x1, one mixed call, every
rejected descriptor writing nothing, and realistic decoder frame sizes."""
import ctypes as C

import numpy as np
import pytest

import oracle
from imageflow_b200 import synth

pytestmark = pytest.mark.gpu

MATTE = (40, 120, 250, 200)


def _ifb():
    import imageflow_b200 as ifb
    return ifb


def _rows_np(iw, ih, bpp, seed, alpha_mode="mixed", content="noise"):
    bgra = synth.cutout_np(iw, ih, seed=seed) if content == "cutout" else synth.noise_np(iw, ih, seed=seed, alpha_mode=alpha_mode)
    return np.ascontiguousarray(bgra[..., [2, 1, 0, 3]][..., :bpp])


def to_bgra(rows):
    h, w, c = rows.shape
    out = np.full((h, w, 4), 255, np.uint8)
    out[..., 0], out[..., 1], out[..., 2] = rows[..., 2], rows[..., 1], rows[..., 0]
    if c == 4:
        out[..., 3] = rows[..., 3]
    return out


def _device_rows(rows, phase=0, pad=0):
    """the rows as a device tensor view `phase` BYTES into a buffer whose rows are `pad` bytes longer than phase + the rows' bytes
    (RGB24 views may start at any byte; RGBA32 phases must be multiples of 4)"""
    import torch
    h, w, c = rows.shape
    pitch = phase + w * c + pad
    buf = torch.zeros(h * pitch + 16, dtype=torch.uint8, device="cuda")
    base = (16 - buf.data_ptr() % 16) % 16                               # pitch phases are relative to a 16-byte aligned address
    flat = np.zeros((h, pitch), np.uint8)
    flat[:, phase:phase + w * c] = rows.reshape(h, w * c)
    buf[base:base + h * pitch] = torch.from_numpy(flat.reshape(-1)).cuda()
    return torch.as_strided(buf, (h, w, c), (pitch, c, 1), base + phase)


def _canvas(cv, compose):
    import torch
    ifb = _ifb()
    t = torch.from_numpy(cv.copy()).cuda()
    return ifb.BitmapWindow.from_torch(t, compose=ifb.BitmapCompositing(compose), matte_bgra=MATTE)


def _params(ow, oh, x, y, filter, linear, sharpen):
    ifb = _ifb()
    return ifb.ScaleAndRenderParams(x=x, y=y, w=ow, h=oh, sharpen_percent_goal=sharpen, interpolation_filter=filter,
                                    scale_in_colorspace=ifb.WorkingFloatspace.LinearRGB if linear else ifb.WorkingFloatspace.StandardRGB)


def _case(b, rows, ow, oh, *, filter=2, linear=True, alpha=None, compose=0, cm=None, sharpen=0.0, phase=0, pad=0, canvas=None, x=0, y=0,
          two_step=True):
    """(fused, two-step, oracle) results of one job, and the (ring kernel, generic pair) job counts of the rows call; alpha None = the
    decoder's choice (RGBA: meaningful)"""
    import torch
    ifb = _ifb()
    am = rows.shape[2] == 4 if alpha is None else alpha
    cv = np.zeros((oh + y + 2, ow + x + 3, 4), np.uint8) if canvas is None else canvas
    src = _device_rows(rows, phase, pad)
    p = _params(ow, oh, x, y, filter, linear, sharpen)
    fused = _canvas(cv, compose)
    f0, g0 = b.fused_jobs, b.generic_jobs
    b.scale_and_render_rows([(src, fused, p, cm, am)], stream="own")
    path = (b.fused_jobs - f0, b.generic_jobs - g0)
    two = None
    if two_step:
        h, w = rows.shape[:2]
        scratch = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
        win = ifb.BitmapWindow.from_torch(scratch)
        b.pixel_convert([ifb.pixel_op_for(rows.shape[2])(src, win)], stream="own")
        win.alpha_meaningful = am
        two = _canvas(cv, compose)
        b.scale_and_render_many([(win, two, p, cm)], stream="own")
    b.sync()
    want = cv.copy()
    oracle.scale_and_render(to_bgra(rows), want, x=x, y=y, w=ow, h=oh, filter=filter, alpha_meaningful=am, linear=linear, compose=compose,
                            matte=MATTE, color_matrix=cm, sharpen=sharpen)
    return fused._keep.cpu().numpy(), (two._keep.cpu().numpy() if two is not None else None), want, path


def _assert_same(got, want, what):
    assert np.array_equal(got, want), (what, np.argwhere(np.any(got != want, axis=2))[:4].tolist())


def _check(b, rows, ow, oh, **kw):
    fused, two, want, path = _case(b, rows, ow, oh, **kw)
    _assert_same(fused, want, ("oracle", rows.shape, ow, oh, kw))
    if two is not None:
        _assert_same(fused, two, ("two-step", rows.shape, ow, oh, kw))
    return path


@pytest.mark.parametrize("bpp", [3, 4])
@pytest.mark.parametrize("force_generic", [0, 1])
def test_both_formats_on_the_ring_kernel_and_the_generic_pair(bpp, force_generic):
    ifb = _ifb()
    b = ifb.Batch(0)
    b.set_option(ifb.Batch.OPT_FORCE_GENERIC, force_generic)
    rows = _rows_np(960, 540, bpp, seed=5)
    for alpha in (False, True):
        assert _check(b, rows, 128, 128, alpha=alpha) == ((0, 1) if force_generic else (1, 0)), (bpp, alpha)
    b.close()


@pytest.mark.parametrize("bpp", [3, 4])
@pytest.mark.parametrize("alpha", [False, True])
@pytest.mark.parametrize("linear", [False, True])
@pytest.mark.parametrize("compose", [0, 1, 2])
def test_store_forms(bpp, alpha, linear, compose):
    """channels x working space x compositing x sharpen x colour matrix, both ring depths, on noise over a mixed-alpha canvas"""
    ifb = _ifb()
    b = ifb.Batch(0)
    rows = _rows_np(704, 500, bpp, seed=7, alpha_mode="mixed" if alpha else "opaque")
    cv = synth.noise_np(260, 260, seed=8, alpha_mode="mixed")
    for cm, sharpen, flt in ((None, 0.0, 2), (ifb.color_filter_matrix(0), 0.0, 6), (None, 40.0, 13), (ifb.color_filter_matrix(3), 0.0, 4)):
        _check(b, rows, 210, 150, alpha=alpha, linear=linear, compose=compose, cm=cm, sharpen=sharpen, filter=flt, canvas=cv, x=7, y=5)
    b.close()


@pytest.mark.parametrize("compose", [0, 1, 2])
def test_cutout_rgba_reaches_the_alpha_branches(compose):
    ifb = _ifb()
    b = ifb.Batch(0)
    rows = _rows_np(640, 480, 4, seed=9, content="cutout")
    cv = synth.cutout_canvas_np(220, 220, seed=3)
    for linear in (True, False):
        path = _check(b, rows, 200, 150, compose=compose, linear=linear, canvas=cv, x=3, y=2, cm=ifb.color_filter_matrix(0) if compose == 2 else None)
        assert path == (1, 0)
    b.close()


def test_rgb24_sub_windows_at_every_byte_phase():
    """RGB24 rows at byte 0..15 of a 16-byte group, with a 16-byte pitch (the ring kernel) and a pitch 1 byte longer (the generic pair)"""
    ifb = _ifb()
    b = ifb.Batch(0)
    rows = _rows_np(333, 277, 3, seed=10)
    for phase in range(16):
        for extra in (0, 1):
            pad = (16 - (phase + 333 * 3) % 16) % 16 + extra
            path = _check(b, rows, 79, 61, phase=phase, pad=pad, alpha=phase % 3 == 0, two_step=phase % 4 == 0)
            assert path == ((1, 0) if extra == 0 else (0, 1)), (phase, extra)
    b.close()


def test_rgba_phases_and_pitches():
    """RGBA32 rows at 4-byte phases of a 16-byte group and padded pitches: only a 16-byte aligned window and pitch take the ring kernel"""
    ifb = _ifb()
    b = ifb.Batch(0)
    rows = _rows_np(333, 277, 4, seed=11)
    for phase in (0, 4, 8, 12):
        for pad in (0, 4, 12, 20):
            path = _check(b, rows, 79, 61, phase=phase, pad=pad, two_step=pad == 0)
            ring = phase == 0 and (333 * 4 + pad) % 16 == 0
            assert path == ((1, 0) if ring else (0, 1)), (phase, pad)
    b.close()


def test_contiguous_tensor_widths():
    """a contiguous (H, W, 3) tensor takes the ring kernel exactly when W is a multiple of 16"""
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    for w in (320, 321, 330, 336):
        rows = _rows_np(w, 200, 3, seed=w)
        t = torch.from_numpy(rows).cuda()
        out = _canvas(np.zeros((50, 80, 4), np.uint8), 0)
        f0 = b.fused_jobs
        b.scale_and_render_rows([(t, out, _params(80, 50, 0, 0, 2, True, 0.0))], stream="own")
        b.sync()
        want = np.zeros((50, 80, 4), np.uint8)
        oracle.scale_and_render(to_bgra(rows), want, w=80, h=50, filter=2, alpha_meaningful=False, linear=True)
        _assert_same(out._keep.cpu().numpy(), want, w)
        assert (b.fused_jobs - f0 == 1) == (w % 16 == 0), w
    b.close()


@pytest.mark.parametrize("bpp", [3, 4])
def test_an_up_scale_and_one_pixel(bpp):
    ifb = _ifb()
    b = ifb.Batch(0)
    for (iw, ih, ow, oh) in ((100, 60, 300, 180), (1, 1, 1, 1), (1, 1, 7, 5), (64, 64, 64, 64)):
        rows = _rows_np(iw, ih, bpp, seed=iw + 6)
        # the generic pair: no ring kernel for up-scales and 1:1, no tile-kernel form
        assert _check(b, rows, ow, oh, alpha=bpp == 4) == (0, 1), (iw, ow)
    b.close()


def test_one_mixed_call_of_both_formats():
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    rng = np.random.default_rng(12)
    jobs, wants, outs = [], [], []
    for i in range(40):
        bpp = int(rng.integers(3, 5))
        iw, ih = int(rng.integers(20, 900)), int(rng.integers(20, 900))
        ow, oh = int(rng.integers(4, 300)), int(rng.integers(4, 300))
        alpha = bool(rng.integers(0, 2))
        rows = _rows_np(iw, ih, bpp, seed=100 + i, alpha_mode="mixed" if alpha else "opaque")
        phase = int(rng.integers(0, 16)) if bpp == 3 else 4 * int(rng.integers(0, 4)) * int(rng.integers(0, 2))
        pad = int(rng.integers(0, 20)) // (4 if bpp == 4 else 1) * (4 if bpp == 4 else 1)
        if rng.integers(0, 2):
            pad = (16 - (phase + iw * bpp) % 16) % 16                  # a 16-byte pitch
        src = _device_rows(rows, phase, pad)
        cv = synth.noise_np(ow + 4, oh + 4, seed=200 + i, alpha_mode="mixed")
        compose = int(rng.integers(0, 3))
        out = _canvas(cv, compose)
        flt = int(rng.choice([2, 6, 13, 14, 24]))
        linear = bool(rng.integers(0, 2))
        cm = ifb.color_filter_matrix(0) if rng.integers(0, 4) == 0 else None
        jobs.append((src, out, _params(ow, oh, 2, 3, flt, linear, 0.0), cm, alpha))
        want = cv.copy()
        oracle.scale_and_render(to_bgra(rows), want, x=2, y=3, w=ow, h=oh, filter=flt, alpha_meaningful=alpha, linear=linear, compose=compose,
                                matte=MATTE, color_matrix=cm)
        wants.append(want); outs.append(out)
    f0, g0 = b.fused_jobs, b.generic_jobs
    b.scale_and_render_rows(jobs, stream="own")
    b.sync()
    assert b.fused_jobs - f0 > 0 and b.generic_jobs - g0 > 0 and (b.fused_jobs - f0) + (b.generic_jobs - g0) == 40
    for i, (out, want) in enumerate(zip(outs, wants)):
        _assert_same(out._keep.cpu().numpy(), want, i)
    torch.cuda.synchronize()
    b.close()


def test_rejected_descriptors_write_nothing():
    import torch
    ifb = _ifb()
    from imageflow_b200._lib import RowsResampleDesc
    b = ifb.Batch(0)
    rows3 = torch.from_numpy(_rows_np(300, 200, 3, seed=15)).cuda()
    rows4 = torch.from_numpy(_rows_np(300, 200, 4, seed=15)).cuda()
    p = _params(60, 40, 0, 0, 2, True, 0.0)
    for bad in ("format2", "format3", "format4", "format-1", "format99", "stride3", "stride4", "misaligned_ptr", "misaligned_stride", "null",
                "rect", "filter"):
        outs = [_canvas(np.full((40, 60, 4), 7, np.uint8), 0) for _ in range(3)]
        descs, keep = b.make_rows_descs([(rows3, outs[0], p), (rows4, outs[1], p), (rows3, outs[2], p)])
        d = descs[1]
        if bad.startswith("format"):
            d.format = int(bad[6:])
            msg = "pixel_convert" if bad in ("format2", "format3") else "is not IFB200_PIXEL_RGB24_TO_BGRA"
        elif bad == "stride3":
            d.format = 0; d.draw.in_stride = 300 * 3 - 1; msg = "smaller than a row of 300 RGB24 pixels"
        elif bad == "stride4":
            d.draw.in_stride = 300 * 4 - 4; msg = "smaller than a row of 300 RGBA32 pixels"
        elif bad == "misaligned_ptr":
            d.draw.in_ = d.draw.in_ + 1; d.draw.in_w = 299; msg = "4-byte aligned"
        elif bad == "misaligned_stride":
            d.draw.in_stride = 300 * 4 + 2; d.draw.in_h = 199; msg = "4-byte aligned"
        elif bad == "null":
            d.draw.in_ = None; msg = "null bitmap pointer"
        elif bad == "rect":
            d.draw.x = 5; msg = "out of bounds"
        else:
            d.draw.filter = 99; msg = "unknown filter id 99"
        with pytest.raises(ifb.FlowError) as e:
            b.enqueue_rows(descs, "own", keep)
        assert f"rows resample job 1: " in str(e.value) and msg in str(e.value), (bad, str(e.value))
        b.sync()
        for o in outs:
            assert (o._keep.cpu().numpy() == 7).all(), bad
    # a BGRA window belongs in scale_and_render_many; the null descriptor array
    win = ifb.BitmapWindow.from_torch(rows4)
    with pytest.raises(ifb.FlowError, match="scale_and_render_many"):
        b.scale_and_render_rows([(win, _canvas(np.zeros((40, 60, 4), np.uint8), 0), p)])
    buf = C.create_string_buffer(256)
    rc = ifb.lib().ifb200_batch_enqueue_rows(b._h, None, 1, b.STREAM_OWN, buf, 256)
    assert rc != 0 and b"null descriptor array" in buf.value
    assert ifb.lib().ifb200_batch_enqueue_rows(b._h, None, 0, b.STREAM_OWN, buf, 256) == 0
    assert C.sizeof(RowsResampleDesc) == C.sizeof(ifb.ResampleDesc) + 8 and RowsResampleDesc.format.offset == C.sizeof(ifb.ResampleDesc)
    b.close()


@pytest.mark.parametrize("iw,ih,bpp,ow,oh", [
    (3840, 2160, 3, 512, 288),              # config 2 from nvJPEG's (H, W, 3) tensor
    (7680, 4320, 3, 512, 288),              # 8K
    (4032, 3024, 3, 512, 384),              # 12 MP sensor frames
    (4032, 3024, 4, 512, 384),
])
def test_realistic_sizes(iw, ih, bpp, ow, oh):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    rows = _rows_np(iw, ih, bpp, seed=16)
    t = torch.from_numpy(rows).cuda()                                   # contiguous: W a multiple of 16, so the ring kernel
    f0 = b.fused_jobs
    out = _canvas(np.zeros((oh, ow, 4), np.uint8), 0)
    b.scale_and_render_rows([(t, out, _params(ow, oh, 0, 0, 2, True, 0.0))], stream="own")
    scratch = b.to_bgra(t, stream="own")
    scratch.alpha_meaningful = bpp == 4
    two = _canvas(np.zeros((oh, ow, 4), np.uint8), 0)
    b.scale_and_render_many([(scratch, two, _params(ow, oh, 0, 0, 2, True, 0.0))], stream="own")
    b.sync()
    want = np.zeros((oh, ow, 4), np.uint8)
    oracle.scale_and_render(to_bgra(rows), want, w=ow, h=oh, filter=2, alpha_meaningful=bpp == 4, linear=True)
    _assert_same(out._keep.cpu().numpy(), want, (iw, ih, bpp))
    _assert_same(out._keep.cpu().numpy(), two._keep.cpu().numpy(), (iw, ih, bpp))
    assert b.fused_jobs - f0 == 2
    b.close()
