"""The oriented rows resample on the GPU (Batch.scale_and_render_rows_oriented -> ifb200_batch_enqueue_rows_oriented), bit for bit
against both the two-step route on the device (Batch.pixel_convert into a BGRA scratch frame, then Batch.scale_and_render_oriented)
and the oracle's scale_and_render of the rows converted and oriented in numpy: every EXIF flag for RGB24 and RGBA32 on the ring
kernel's oriented row forms and on the generic pair (the counters confirm which ran), widths that are not a multiple of four, the
store forms, cut-out alpha, RGB24 windows at every byte phase, up-scales, 1:1 and 1x1, identity flags running exactly as
scale_and_render_rows, one mixed call, a crop through oriented_source_rect, every rejected descriptor writing nothing, the struct
layout, realistic photo sizes and an oriented frame taller than one grid on the generic H pass."""
import ctypes as C

import numpy as np
import pytest

import oracle
from imageflow_b200 import synth
from tests import orient_oracle
from tests.test_rows_resample_gpu import MATTE, _assert_same, _canvas, _device_rows, _ifb, _params, _rows_np, to_bgra

pytestmark = pytest.mark.gpu


def _case(b, rows, ow, oh, flag, *, filter=2, linear=True, alpha=None, compose=0, cm=None, sharpen=0.0, phase=0, pad=0, canvas=None, x=0,
          y=0, two_step=True):
    """(fused, two-step, oracle) results of one job, and the (ring kernel, generic pair) job counts of the oriented rows call; alpha
    None = the decoder's choice (RGBA: meaningful)"""
    import torch
    ifb = _ifb()
    am = rows.shape[2] == 4 if alpha is None else alpha
    cv = np.zeros((oh + y + 2, ow + x + 3, 4), np.uint8) if canvas is None else canvas
    src = _device_rows(rows, phase, pad)
    p = _params(ow, oh, x, y, filter, linear, sharpen)
    fused = _canvas(cv, compose)
    f0, g0 = b.fused_jobs, b.generic_jobs
    b.scale_and_render_rows_oriented([(src, fused, p, flag, cm, am)], stream="own")
    path = (b.fused_jobs - f0, b.generic_jobs - g0)
    two = None
    if two_step:
        h, w = rows.shape[:2]
        scratch = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
        win = ifb.BitmapWindow.from_torch(scratch)
        b.pixel_convert([ifb.pixel_op_for(rows.shape[2])(src, win)], stream="own")
        win.alpha_meaningful = am
        two = _canvas(cv, compose)
        b.scale_and_render_oriented([(win, two, p, flag, cm)], stream="own")
    b.sync()
    want = cv.copy()
    oracle.scale_and_render(np.ascontiguousarray(orient_oracle.gather(to_bgra(rows), flag)), want, x=x, y=y, w=ow, h=oh, filter=filter,
                            alpha_meaningful=am, linear=linear, compose=compose, matte=MATTE, color_matrix=cm, sharpen=sharpen)
    return fused._keep.cpu().numpy(), (two._keep.cpu().numpy() if two is not None else None), want, path


def _check(b, rows, ow, oh, flag, **kw):
    fused, two, want, path = _case(b, rows, ow, oh, flag, **kw)
    _assert_same(fused, want, ("oracle", rows.shape, ow, oh, flag, kw))
    if two is not None:
        _assert_same(fused, two, ("two-step", rows.shape, ow, oh, flag, kw))
    return path


def _aligned(rows):
    """the device rows with a pitch that is a multiple of 16 bytes (the ring kernel's rule for both formats)"""
    h, w, c = rows.shape
    return dict(pad=(16 - (w * c) % 16) % 16)


@pytest.mark.parametrize("bpp", [3, 4])
@pytest.mark.parametrize("force_generic", [0, 1])
def test_every_flag_on_the_ring_kernel_and_the_generic_pair(bpp, force_generic):
    ifb = _ifb()
    b = ifb.Batch(0)
    b.set_option(ifb.Batch.OPT_FORCE_GENERIC, force_generic)
    rows = _rows_np(960, 540, bpp, seed=5)
    for flag in range(-1, 10):
        for alpha in (False, True):
            path = _check(b, rows, 128, 128, flag, alpha=alpha, two_step=alpha == (flag % 2 == 0))
            assert path == ((0, 1) if force_generic else (1, 0)), (bpp, flag, alpha)
    b.close()


@pytest.mark.parametrize("bpp", [3, 4])
def test_widths_not_a_multiple_of_four(bpp):
    """source x reversed (flags 2, 3, 7, 8): RGB24 keeps the ring kernel at any width; RGBA32 keeps the BGRA rule and takes the
    generic pair"""
    ifb = _ifb()
    b = ifb.Batch(0)
    for iw in (961, 962, 963):
        rows = _rows_np(iw, 541, bpp, seed=iw)
        for flag in (2, 3, 4, 6, 7, 8):
            path = _check(b, rows, 128, 128, flag, **_aligned(rows), two_step=flag in (3, 8))
            ring = bpp == 3 or flag not in (2, 3, 7, 8)
            assert path == ((1, 0) if ring else (0, 1)), (bpp, iw, flag)
    b.close()


@pytest.mark.parametrize("bpp", [3, 4])
@pytest.mark.parametrize("alpha", [False, True])
@pytest.mark.parametrize("linear", [False, True])
@pytest.mark.parametrize("compose", [0, 1, 2])
def test_store_forms(bpp, alpha, linear, compose):
    """channels x working space x compositing x sharpen x colour matrix, both ring depths, flips and transposes"""
    ifb = _ifb()
    b = ifb.Batch(0)
    rows = _rows_np(704, 500, bpp, seed=7, alpha_mode="mixed" if alpha else "opaque")
    cv = synth.noise_np(260, 260, seed=8, alpha_mode="mixed")
    for flag, cm, sharpen, flt in ((6, None, 0.0, 2), (3, ifb.color_filter_matrix(0), 0.0, 6), (8, None, 40.0, 13),
                                   (2, ifb.color_filter_matrix(3), 0.0, 4), (7, ifb.color_filter_matrix(0), 30.0, 6)):
        _check(b, rows, 210, 150, flag, alpha=alpha, linear=linear, compose=compose, cm=cm, sharpen=sharpen, filter=flt, canvas=cv, x=7, y=5,
               two_step=flag in (6, 7))
    b.close()


@pytest.mark.parametrize("compose", [0, 1, 2])
def test_cutout_rgba_reaches_the_alpha_branches(compose):
    ifb = _ifb()
    b = ifb.Batch(0)
    rows = _rows_np(640, 480, 4, seed=9, content="cutout")
    cv = synth.cutout_canvas_np(220, 220, seed=3)
    for flag in (3, 6, 8):
        path = _check(b, rows, 200, 150, flag, compose=compose, canvas=cv, x=3, y=2, cm=ifb.color_filter_matrix(0) if compose == 2 else None)
        assert path == (1, 0), flag
    b.close()


def test_rgb24_windows_at_every_byte_phase():
    """RGB24 rows at byte 0..15 of a 16-byte group, under reversed and transposed reads, with a 16-byte pitch (the ring kernel) and
    a pitch 1 byte longer (the generic pair)"""
    ifb = _ifb()
    b = ifb.Batch(0)
    rows = _rows_np(333, 277, 3, seed=10)
    for phase in range(16):
        for extra in (0, 1):
            pad = (16 - (phase + 333 * 3) % 16) % 16 + extra
            for flag in ((2, 7) if phase % 2 else (3, 6, 8)):
                path = _check(b, rows, 79, 61, flag, phase=phase, pad=pad, alpha=phase % 3 == 0, two_step=phase % 4 == 0)
                assert path == ((1, 0) if extra == 0 else (0, 1)), (phase, extra, flag)
    b.close()


@pytest.mark.parametrize("bpp", [3, 4])
def test_an_up_scale_one_to_one_and_one_pixel(bpp):
    ifb = _ifb()
    b = ifb.Batch(0)
    for (iw, ih, ow, oh) in ((100, 60, 180, 300), (1, 1, 1, 1), (1, 1, 7, 5), (64, 64, 64, 64), (3, 2, 9, 4)):
        rows = _rows_np(iw, ih, bpp, seed=iw + 6)
        for flag in (3, 6, 8):
            assert _check(b, rows, ow, oh, flag, alpha=bpp == 4) == (0, 1), (iw, ow, flag)
    b.close()


@pytest.mark.parametrize("bpp", [3, 4])
def test_identity_flags_run_as_scale_and_render_rows(bpp):
    """flags 1, 0, -1 and 9: the same kernel, bytes and counters as scale_and_render_rows, on the ring kernel and the generic pair"""
    ifb = _ifb()
    b = ifb.Batch(0)
    for (iw, ih, ow, oh, pad) in ((960, 540, 128, 128, 0), (333, 277, 79, 61, 1), (100, 60, 300, 180, 0)):
        rows = _rows_np(iw, ih, bpp, seed=iw)
        pad = pad * (4 if bpp == 4 else 1) + (16 - (iw * bpp) % 16) % 16
        src = _device_rows(rows, 0, pad)
        p = _params(ow, oh, 1, 2, 2, True, 0.0)
        cv = synth.noise_np(ow + 4, oh + 4, seed=3, alpha_mode="mixed")
        plain = _canvas(cv, 1)
        c0 = (b.fused_jobs, b.generic_jobs, b.kernel_launches)
        b.scale_and_render_rows([(src, plain, p)], stream="own")
        c1 = (b.fused_jobs, b.generic_jobs, b.kernel_launches)
        moved = tuple(u - v for u, v in zip(c1, c0))                   # what the rows call moved the counters by
        for flag in (1, 0, -1, 9):
            out = _canvas(cv, 1)
            b.scale_and_render_rows_oriented([(src, out, p, flag)], stream="own")
            c2 = (b.fused_jobs, b.generic_jobs, b.kernel_launches)
            assert tuple(u - v for u, v in zip(c2, c1)) == moved, (iw, flag)
            c1 = c2
            b.sync()
            _assert_same(out._keep.cpu().numpy(), plain._keep.cpu().numpy(), (iw, flag))
    b.close()


def test_one_mixed_call_of_both_formats_and_every_flag():
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    rng = np.random.default_rng(12)
    jobs, wants, outs = [], [], []
    for i in range(40):
        bpp = int(rng.integers(3, 5))
        flag = int(rng.integers(0, 10))
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
        jobs.append((src, out, _params(ow, oh, 2, 3, flt, linear, 0.0), flag, cm, alpha))
        want = cv.copy()
        oracle.scale_and_render(np.ascontiguousarray(orient_oracle.gather(to_bgra(rows), flag)), want, x=2, y=3, w=ow, h=oh, filter=flt,
                                alpha_meaningful=alpha, linear=linear, compose=compose, matte=MATTE, color_matrix=cm)
        wants.append(want); outs.append(out)
    f0, g0 = b.fused_jobs, b.generic_jobs
    b.scale_and_render_rows_oriented(jobs, stream="own")
    b.sync()
    assert b.fused_jobs - f0 > 0 and b.generic_jobs - g0 > 0 and (b.fused_jobs - f0) + (b.generic_jobs - g0) == 40
    for i, (out, want) in enumerate(zip(outs, wants)):
        _assert_same(out._keep.cpu().numpy(), want, (i, jobs[i][3]))
    torch.cuda.synchronize()
    b.close()


def test_a_crop_through_oriented_source_rect():
    """a crop of the oriented frame is a slice of the rows tensor at oriented_source_rect, the rectangle oriented_source_window takes"""
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    rows = _rows_np(640, 480, 3, seed=21)
    t = torch.from_numpy(rows).cuda()
    for flag in range(1, 9):
        x1, y1, x2, y2 = 30, 17, 401, 290
        sx1, sy1, sx2, sy2 = ifb.oriented_source_rect(640, 480, flag, x1, y1, x2, y2)
        win = ifb.oriented_source_window(ifb.BitmapWindow(0, 640, 480, 640 * 4), flag, x1, y1, x2, y2)
        assert (win.ptr // 4 % 640, win.ptr // 4 // 640, win.w, win.h) == (sx1, sy1, sx2 - sx1, sy2 - sy1), flag
        out = _canvas(np.zeros((60, 90, 4), np.uint8), 0)
        b.scale_and_render_rows_oriented([(t[sy1:sy2, sx1:sx2], out, _params(90, 60, 0, 0, 2, True, 0.0), flag)], stream="own")
        b.sync()
        want = np.zeros((60, 90, 4), np.uint8)
        crop = np.ascontiguousarray(orient_oracle.gather(to_bgra(rows), flag)[y1:y2, x1:x2])
        oracle.scale_and_render(crop, want, w=90, h=60, filter=2, alpha_meaningful=False, linear=True)
        _assert_same(out._keep.cpu().numpy(), want, flag)
    assert ifb.oriented_source_rect(640, 480, 6, 0, 0, 481, 10) is None
    b.close()


def test_rejected_descriptors_write_nothing():
    import torch
    ifb = _ifb()
    from imageflow_b200._lib import RowsOrientedResampleDesc
    b = ifb.Batch(0)
    rows3 = torch.from_numpy(_rows_np(300, 200, 3, seed=15)).cuda()
    rows4 = torch.from_numpy(_rows_np(300, 200, 4, seed=15)).cuda()
    p = _params(60, 40, 0, 0, 2, True, 0.0)
    for bad in ("format2", "format3", "format4", "format-1", "format99", "stride3", "stride4", "misaligned_ptr", "misaligned_stride", "null",
                "rect", "filter"):
        outs = [_canvas(np.full((40, 60, 4), 7, np.uint8), 0) for _ in range(3)]
        descs, keep = b.make_rows_oriented_descs([(rows3, outs[0], p, 6), (rows4, outs[1], p, 8), (rows3, outs[2], p, 1)])
        d = descs[1]
        if bad.startswith("format"):
            d.format = int(bad[6:])
            msg = "ifb200_batch_enqueue_oriented" if bad in ("format2", "format3") else "is not IFB200_PIXEL_RGB24_TO_BGRA"
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
            b.enqueue_rows_oriented(descs, "own", keep)
        assert "oriented rows resample job 1: " in str(e.value) and msg in str(e.value), (bad, str(e.value))
        b.sync()
        for o in outs:
            assert (o._keep.cpu().numpy() == 7).all(), bad
    win = ifb.BitmapWindow.from_torch(rows4)
    with pytest.raises(ifb.FlowError, match="scale_and_render_oriented"):
        b.scale_and_render_rows_oriented([(win, _canvas(np.zeros((40, 60, 4), np.uint8), 0), p, 6)])
    buf = C.create_string_buffer(256)
    rc = ifb.lib().ifb200_batch_enqueue_rows_oriented(b._h, None, 1, b.STREAM_OWN, buf, 256)
    assert rc != 0 and b"null descriptor array" in buf.value
    assert ifb.lib().ifb200_batch_enqueue_rows_oriented(b._h, None, 0, b.STREAM_OWN, buf, 256) == 0
    b.close()


def test_struct_layout():
    ifb = _ifb()
    from imageflow_b200._lib import RowsOrientedResampleDesc
    n = C.sizeof(ifb.ResampleDesc)
    assert RowsOrientedResampleDesc.format.offset == n and RowsOrientedResampleDesc.orientation.offset == n + 4
    assert C.sizeof(RowsOrientedResampleDesc) == n + 8


@pytest.mark.parametrize("iw,ih,bpp,flag,ow,oh,content", [
    (4032, 3024, 3, 6, 384, 512, "noise"),  # a portrait phone photo from nvJPEG's (H, W, 3) tensor
    (4032, 3024, 3, 8, 384, 512, "noise"),
    (3840, 2160, 3, 3, 512, 288, "noise"),  # upside down 4K
    (7680, 4320, 4, 8, 288, 512, "cutout"),  # 8K RGBA32
])
def test_realistic_sizes(iw, ih, bpp, flag, ow, oh, content):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    rows = _rows_np(iw, ih, bpp, seed=16, content=content)
    t = torch.from_numpy(rows).cuda()                                   # contiguous: W a multiple of 16, so the ring kernel
    f0 = b.fused_jobs
    out = _canvas(np.zeros((oh, ow, 4), np.uint8), 0)
    b.scale_and_render_rows_oriented([(t, out, _params(ow, oh, 0, 0, 2, True, 0.0), flag)], stream="own")
    scratch = b.to_bgra(t, stream="own")
    scratch.alpha_meaningful = bpp == 4
    two = _canvas(np.zeros((oh, ow, 4), np.uint8), 0)
    b.scale_and_render_oriented([(scratch, two, _params(ow, oh, 0, 0, 2, True, 0.0), flag)], stream="own")
    b.sync()
    want = np.zeros((oh, ow, 4), np.uint8)
    oracle.scale_and_render(np.ascontiguousarray(orient_oracle.gather(to_bgra(rows), flag)), want, w=ow, h=oh, filter=2, alpha_meaningful=bpp == 4,
                            linear=True)
    _assert_same(out._keep.cpu().numpy(), want, (iw, ih, bpp, flag))
    _assert_same(out._keep.cpu().numpy(), two._keep.cpu().numpy(), (iw, ih, bpp, flag))
    assert b.fused_jobs - f0 == 2
    b.close()


@pytest.mark.parametrize("bpp", [3, 4])
def test_oriented_height_beyond_one_grid_on_the_generic_h_pass(bpp):
    """an oriented frame 70 000 rows tall: stored 70 000 x 4 with flag 6 (threads along a source row, output columns on grid y) and
    stored 4 x 70 000 with flag 3 (oriented rows on grid y, walked past 65 535)"""
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    b.set_option(ifb.Batch.OPT_FORCE_GENERIC, 1)
    for (iw, ih, flag) in ((70000, 4, 6), (4, 70000, 3)):
        rows = _rows_np(iw, ih, bpp, seed=iw % 97)
        t = torch.from_numpy(rows).cuda()
        out = _canvas(np.zeros((35000, 3, 4), np.uint8), 0)
        l0, g0 = b.kernel_launches, b.generic_jobs
        b.scale_and_render_rows_oriented([(t, out, _params(3, 35000, 0, 0, 2, True, 0.0), flag)], stream="own")
        b.sync()
        assert (b.kernel_launches - l0, b.generic_jobs - g0) == (2, 1), flag
        want = np.zeros((35000, 3, 4), np.uint8)
        oracle.scale_and_render(np.ascontiguousarray(orient_oracle.gather(to_bgra(rows), flag)), want, w=3, h=35000, filter=2,
                                alpha_meaningful=bpp == 4, linear=True)
        _assert_same(out._keep.cpu().numpy(), want, (iw, ih, flag))
    b.close()
