"""Pixel-format conversions on the GPU (pixel_convert_kernel through Batch.pixel_convert), bit for bit against
tests/pixel_convert_oracle.py: every op with and without opaque on 1x1, odd sizes, 4K and 8K, padded strides and sub-windows with
sentinel bytes around them; the emulation's multi-job launches at every phase; batches of 1, 7 and 64 jobs as one launch and a call
with nothing to write as none; a bad descriptor that changes nothing; a (2160, 3840, 3) CUDA tensor into BGRA and through the config-2
resample against the oracle; and a resampled frame out to RGB24 and to opaque RGBA."""
import numpy as np
import pytest

import oracle
from tests import pixel_convert_oracle as po
from tests.cpu_emu import run_pixel_convert_cases as rpc

pytestmark = pytest.mark.gpu


def _ifb():
    import imageflow_b200 as ifb
    return ifb


def _rows(t, x, y, w, h):
    """the (h, w, C) sub-window at (x, y) of a (H, W, C) tensor, as PixelRows"""
    return _ifb().PixelRows.from_torch(t[y:y + h, x:x + w])


def _job(op, src, dst, opaque):
    return _ifb().graphics._PIXEL_OPS[op](src, dst, opaque)


SIZES = [(1, 1), (3, 1), (1, 5), (17, 9), (33, 7), (101, 13), (3840, 2160), (7680, 4320)]


@pytest.mark.parametrize("op", po.OPS)
@pytest.mark.parametrize("opaque", [False, True])
def test_every_op_on_sub_windows_of_padded_bitmaps(op, opaque):
    """each size as a sub-window at an odd origin of a bitmap with padded rows, sentinel bytes all around; all sizes in one call"""
    import torch
    ifb = _ifb()
    cs, cd = po.CHANNELS[op]
    rng = np.random.default_rng(7 + op)
    jobs, checks = [], []
    for i, (w, h) in enumerate(SIZES):
        sx, sy, dx, dy = 1 + i % 3, 2, (i + 1) % 4, 1
        src = rng.integers(0, 256, (h + 3, w + 5, cs), dtype=np.uint8)
        dst = rng.integers(0, 256, (h + 2, w + 7, cd), dtype=np.uint8)
        ts, td = torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda()
        jobs.append(_job(op, _rows(ts, sx, sy, w, h), _rows(td, dx, dy, w, h), opaque))
        want = dst.copy()
        want[dy:dy + h, dx:dx + w] = po.convert(op, src[sy:sy + h, sx:sx + w], opaque)
        checks.append((td, want, src, ts))
    b = ifb.Batch(0)
    n0 = b.kernel_launches
    b.pixel_convert(jobs, stream="own")
    b.sync()
    assert b.kernel_launches == n0 + 1
    for (td, want, src, ts), size in zip(checks, SIZES):
        got = td.cpu().numpy()
        assert np.array_equal(got, want), (size, np.argwhere(got != want)[:4].tolist())
        assert np.array_equal(ts.cpu().numpy(), src), size


def test_in_place_swap_with_and_without_opaque():
    import torch
    ifb = _ifb()
    rng = np.random.default_rng(3)
    b = ifb.Batch(0)
    for opaque in (False, True):
        for (w, h) in [(1, 1), (7, 3), (3840, 2160)]:
            a = rng.integers(0, 256, (h + 2, w + 3, 4), dtype=np.uint8)
            t = torch.from_numpy(a).cuda()
            win = ifb.BitmapWindow.from_torch(t[1:1 + h, 1:1 + w])
            out = b.pixel_convert([ifb.RgbaToBgra(win, None, opaque)], stream="own")
            b.sync()
            want = a.copy()
            want[1:1 + h, 1:1 + w] = po.convert(po.RGBA_TO_BGRA, a[1:1 + h, 1:1 + w], opaque)
            assert np.array_equal(t.cpu().numpy(), want), (w, h, opaque)
            assert out[0] is win and win.alpha_meaningful == (not opaque)


def test_the_emulation_launches_on_the_device():
    """the multi-job launches of the CPU emulation (every source phase modulo 16, every destination phase, widths 1..40, in place)"""
    import torch
    ifb = _ifb()
    rng = np.random.default_rng(11)
    b = ifb.Batch(0)
    for jobs in rpc.fixed_launches(rng) + [[rpc.make_job(rng) for _ in range(8)] for _ in range(20)]:
        dev = {id(r): torch.from_numpy(r.buf.copy()).cuda() for _, rs, _, _ in jobs for r in rs}
        recs = []
        for d, rs, _, _ in jobs:
            ptr = lambda r, p: dev[id(r)].data_ptr() + (p - r.buf.ctypes.data)
            s = ifb.PixelRows(ptr(rs[0], d["src"]), d["w"], d["h"], d["src_stride"], rs[0].ch, dev[id(rs[0])])
            t = s if len(rs) == 1 else ifb.PixelRows(ptr(rs[1], d["dst"]), d["w"], d["h"], d["dst_stride"], rs[1].ch, dev[id(rs[1])])
            recs.append(_job(d["op"], s, None if len(rs) == 1 else t, bool(d["opaque"])))
        b.pixel_convert(recs, stream="own")
        b.sync()
        for _, rs, _, _ in jobs:
            for r in rs:
                got = dev[id(r)].cpu().numpy()
                assert np.array_equal(got, r.exp), ([j[0] for j in jobs], np.nonzero(got != r.exp)[0][:4].tolist())


@pytest.mark.parametrize("n", [1, 7, 64])
def test_a_batch_is_one_launch(n):
    import torch
    ifb = _ifb()
    rng = np.random.default_rng(n)
    srcs = [torch.from_numpy(rng.integers(0, 256, (37 + i, 53 + i, 3), dtype=np.uint8)).cuda() for i in range(n)]
    b = ifb.Batch(0)
    n0 = b.kernel_launches
    outs = [torch.zeros((37 + i, 53 + i, 4), dtype=torch.uint8, device="cuda") for i in range(n)]
    b.pixel_convert([ifb.RgbToBgra(s, o) for s, o in zip(srcs, outs)], stream="own")
    b.sync()
    assert b.kernel_launches == n0 + 1
    for s, o in zip(srcs, outs):
        assert np.array_equal(o.cpu().numpy(), po.convert(po.RGB24_TO_BGRA, s.cpu().numpy()))


def test_nothing_to_write_launches_nothing():
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    n0 = b.kernel_launches
    t = torch.zeros((4, 0, 3), dtype=torch.uint8, device="cuda")
    b.pixel_convert([], stream="own")
    b.pixel_convert([ifb.RgbToBgra(t, torch.zeros((4, 0, 4), dtype=torch.uint8, device="cuda"))], stream="own")
    b.sync()
    assert b.kernel_launches == n0


def test_a_bad_descriptor_changes_nothing():
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    src = torch.full((8, 8, 4), 7, dtype=torch.uint8, device="cuda")
    dst = torch.full((8, 8, 4), 9, dtype=torch.uint8, device="cuda")
    n0 = b.kernel_launches
    with pytest.raises(ifb.FlowError) as e:        # the second job's destination overlaps its source
        b.pixel_convert([ifb.RgbaToBgra(src, dst), ifb.RgbaToBgra(_rows(src, 0, 0, 4, 4), _rows(src, 1, 1, 4, 4))], stream="own")
    b.sync()
    assert e.value.kind == ifb.ErrorKind.InvalidArgument and "pixel convert job 1" in str(e.value)
    assert b.kernel_launches == n0 and bool((src == 7).all()) and bool((dst == 9).all())


def test_an_rgb_tensor_into_bgra_then_the_config_2_resample_equals_the_oracle():
    """a (2160, 3840, 3) uint8 CUDA tensor (a GPU decoder's interleaved RGB) into BGRA in one call, then 3840x2160 -> 512x288 Robidoux
    in linear light: against the oracle's resample of the numpy conversion"""
    import torch
    ifb = _ifb()
    rgb = np.random.default_rng(21).integers(0, 256, (2160, 3840, 3), dtype=np.uint8)
    mid = po.convert(po.RGB24_TO_BGRA, rgb)
    want = np.zeros((288, 512, 4), np.uint8)
    oracle.scale_and_render(mid, want, filter=2, linear=True, alpha_meaningful=False)
    b = ifb.Batch(0)
    win = b.to_bgra(torch.from_numpy(rgb).cuda(), stream="own")
    assert (win.w, win.h, win.stride % 64, win.alpha_meaningful) == (3840, 2160, 0, False)
    out = torch.zeros((288, 512, 4), dtype=torch.uint8, device="cuda")
    b.scale_and_render_many([(win, ifb.BitmapWindow.from_torch(out), ifb.ScaleAndRenderParams(w=512, h=288))], stream="own")
    b.sync()
    assert np.array_equal(win._keep.cpu().numpy(), mid)
    got = out.cpu().numpy()
    assert np.array_equal(got, want), np.argwhere(np.any(got != want, axis=2))[:4].tolist()


def test_a_resampled_frame_out_to_rgb24_and_opaque_rgba_equals_numpy():
    import torch
    ifb = _ifb()
    inp = oracle.synth_noise(1920, 1080, seed=5, alpha_mode="mixed")
    b = ifb.Batch(0)
    src = torch.from_numpy(inp).cuda()
    out = torch.zeros((301, 533, 4), dtype=torch.uint8, device="cuda")
    frame = ifb.BitmapWindow.from_torch(out)
    b.scale_and_render_many([(ifb.BitmapWindow.from_torch(src, alpha_meaningful=True), frame, ifb.ScaleAndRenderParams(w=533, h=301))],
                            stream="own")
    rgb = b.from_bgra(frame, 3, stream="own")
    rgba = b.from_bgra(frame, 4, opaque=True, stream="own")
    b.sync()
    f = out.cpu().numpy()
    assert np.array_equal(rgb.cpu().numpy(), f[..., [2, 1, 0]])
    want = f[..., [2, 1, 0, 3]].copy()
    want[..., 3] = 255
    assert np.array_equal(rgba.cpu().numpy(), want)
