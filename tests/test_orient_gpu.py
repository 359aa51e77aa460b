"""Orientation on the GPU (orient_kernel through Batch.orient), bit for bit: every flag in place and out of place on sizes that
straddle the tile, 4K and 8K frames, padded strides and sub-windows with sentinel bytes around them; mixed batches as one launch and
a call with nothing to write as none; a bad descriptor that changes nothing; each flag against the reference's expansion done on the
device with the existing transpose and flip calls; autorotate + srotate + sflip in one call; and flag 6 followed by the config-2
resample against the oracle."""
import numpy as np
import pytest

import oracle
from tests import orient_oracle as oo
from tests.cpu_emu import run_orient_cases as roc

pytestmark = pytest.mark.gpu


def _ifb():
    import imageflow_b200 as ifb
    return ifb


def _upload(jobs):
    import torch
    return {id(b): torch.from_numpy(b.buf.copy()).cuda() for _, bms, _, _ in jobs for b in bms}


def _jobs_of(jobs, dev):
    """Batch.orient jobs for the emulation's job dicts, on device copies `dev` (id(bitmap) -> tensor) of their bitmaps"""
    ifb = _ifb()
    out = []
    for d, bms, _, _ in jobs:
        src = bms[0]
        t = d["orientation"] in (5, 6, 7, 8)
        inp = ifb.BitmapWindow(dev[id(src)].data_ptr() + (d["in_"] - src.buf.ctypes.data), d["in_w"], d["in_h"], d["in_stride"], _keep=dev[id(src)])
        if len(bms) == 1:
            out.append((inp, None, d["orientation"]))
        else:
            dst = bms[1]
            ow, oh = (d["in_h"], d["in_w"]) if t else (d["in_w"], d["in_h"])
            out.append((inp, ifb.BitmapWindow(dev[id(dst)].data_ptr() + (d["out"] - dst.buf.ctypes.data), ow, oh, d["out_stride"],
                                              _keep=dev[id(dst)]), d["orientation"]))
    return out


def _check(jobs, dev, what):
    for _, bms, _, _ in jobs:
        for bm in bms:
            got = dev[id(bm)].cpu().numpy()
            assert np.array_equal(got, bm.exp), (what, np.nonzero(got != bm.exp)[0][:4].tolist())


def test_every_flag_in_place_and_out_of_place_on_straddling_sizes():
    ifb = _ifb()
    b = ifb.Batch(0)
    rng = np.random.default_rng(31)
    for size in roc.SIZES:
        jobs = [roc.make_job(rng, o, ip, size) for o in list(range(1, 9)) + [0, 9, -1] for ip in ((False, True) if o not in (5, 6, 7, 8) else (False,))]
        dev = _upload(jobs)
        b.orient(_jobs_of(jobs, dev), stream="own")
        b.sync()
        _check(jobs, dev, size)


def test_mixed_batches_are_one_launch():
    ifb = _ifb()
    b = ifb.Batch(0)
    rng = np.random.default_rng(32)
    for n in (1, 7, 64):
        for rep in range(3):
            jobs = roc.make_launch(rng, n)
            writes = any(st for _, _, _, st in jobs)
            dev = _upload(jobs)
            before = b.kernel_launches
            b.orient(_jobs_of(jobs, dev), stream="own")
            b.sync()
            assert b.kernel_launches == before + (1 if writes else 0), (n, rep)
            _check(jobs, dev, (n, rep))


def test_call_with_nothing_to_write_launches_nothing():
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    t = torch.full((8, 8, 4), 7, dtype=torch.uint8, device="cuda")
    win = ifb.BitmapWindow.from_torch(t)
    empty = ifb.BitmapWindow(0, 0, 5, 0)
    before = b.kernel_launches
    out = b.orient([(win, None, 1), (win, None, 0), (win, None, 9), (empty, None, 3), (ifb.BitmapWindow(0, 3, 0, 0), None, 2)], stream="own")
    b.orient([], stream="own")
    b.sync()
    assert b.kernel_launches == before and out[0] is win
    assert (t.cpu().numpy() == 7).all()


def test_a_bad_descriptor_changes_nothing_and_launches_nothing():
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    rng = np.random.default_rng(33)
    jobs = roc.make_launch(rng, 7)
    dev = _upload(jobs)
    good = _jobs_of(jobs, dev)
    sq = ifb.BitmapWindow.from_torch(torch.zeros((6, 6, 4), dtype=torch.uint8, device="cuda"))
    over = torch.zeros((8, 16, 4), dtype=torch.uint8, device="cuda")
    for bad in ((sq, None, 6), (sq, sq, 5),                                          # in-place transposes
                (ifb.BitmapWindow.from_torch(over[:, :8]), ifb.BitmapWindow.from_torch(over[:, 4:12]), 2),   # overlapping windows
                (ifb.BitmapWindow(sq.ptr + 2, 6, 6, 24, _keep=sq._keep), None, 2)):      # misaligned
        before = b.kernel_launches
        with pytest.raises(ifb.FlowError) as e:
            b.orient(good[:3] + [bad] + good[3:], stream="own")
        b.sync()
        assert e.value.kind == ifb.ErrorKind.InvalidArgument and "orient job 3" in str(e.value)
        assert b.kernel_launches == before
        for _, bms, _, _ in jobs:
            for bm in bms:
                assert np.array_equal(dev[id(bm)].cpu().numpy(), bm.buf)


def _expansion_on_device(b, t, flag):
    """the reference's expansion of ApplyOrientation(flag) on the device, node by node with the existing single-window calls;
    returns the resulting tensor"""
    import torch
    ifb = _ifb()
    for p in oo.primitives([("ApplyOrientation", flag)]):
        if p == oo.FLIP_H:
            b.flip_horizontal(ifb.BitmapWindow.from_torch(t), stream="own")
        elif p == oo.FLIP_V:
            b.flip_vertical(ifb.BitmapWindow.from_torch(t), stream="own")
        else:
            o = torch.empty((t.shape[1], t.shape[0], 4), dtype=torch.uint8, device="cuda")
            b.transpose(ifb.BitmapWindow.from_torch(t), ifb.BitmapWindow.from_torch(o), stream="own")
            t = o
    return t


@pytest.mark.parametrize("w,h", [(3840, 2160), (7680, 4320)])
@pytest.mark.parametrize("flag", range(1, 9))
def test_4k_and_8k_frames_equal_the_expansion_on_the_device(w, h, flag):
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    host = np.random.default_rng(w + flag).integers(0, 256, (h, w, 4), dtype=np.uint8)
    src = torch.from_numpy(host).cuda()
    want = _expansion_on_device(b, src.clone(), flag)
    job = ifb.apply_orientation(ifb.BitmapWindow.from_torch(src, alpha_meaningful=True), flag)
    out = b.orient([job], stream="own")[0]
    b.sync()
    assert out.alpha_meaningful and (out.w, out.h) == (want.shape[1], want.shape[0])
    assert torch.equal(out._keep, want)
    assert torch.equal(src, torch.from_numpy(host).cuda())               # the input is read only
    if flag in (2, 3, 4):                                                # in place
        b.orient([(ifb.BitmapWindow.from_torch(src), None, flag)], stream="own")
        b.sync()
        assert torch.equal(src, want)
    if w == 3840:                                                        # against the oracle's closed form too
        assert np.array_equal(out._keep.cpu().numpy(), oo.gather(host, flag))


@pytest.mark.parametrize("flag", range(1, 9))
def test_padded_strides_and_sub_windows_keep_their_surroundings(flag):
    """a 1001 x 517 sub-window at (3, 5) of a bitmap with a padded stride, into a sub-window of another; every byte around the two
    windows stays"""
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    rng = np.random.default_rng(40 + flag)
    w, h = 1001, 517
    t = flag >= 5
    ow, oh = (h, w) if t else (w, h)
    src_h = rng.integers(0, 256, (h + 9, w + 13, 4), dtype=np.uint8)
    dst_h = rng.integers(0, 256, (oh + 7, ow + 11, 4), dtype=np.uint8)
    src, dst = torch.from_numpy(src_h).cuda(), torch.from_numpy(dst_h).cuda()
    sw = ifb.BitmapWindow.from_torch(src).window(3, 5, 3 + w, 5 + h)
    dw = ifb.BitmapWindow.from_torch(dst).window(6, 2, 6 + ow, 2 + oh)
    b.orient([(sw, dw, flag)], stream="own")
    b.sync()
    want = dst_h.copy()
    want[2:2 + oh, 6:6 + ow] = oo.gather(src_h[5:5 + h, 3:3 + w], flag)
    assert np.array_equal(dst.cpu().numpy(), want) and np.array_equal(src.cpu().numpy(), src_h)
    if not t:                                                           # in place
        b.orient([(sw, None, flag)], stream="own")
        b.sync()
        want = src_h.copy()
        want[5:5 + h, 3:3 + w] = oo.gather(src_h[5:5 + h, 3:3 + w], flag)
        assert np.array_equal(src.cpu().numpy(), want)


def test_autorotate_srotate_sflip_in_one_call_equals_the_chain():
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    steps = [ifb.ApplyOrientation(6)] + ifb.riapi_rotate_steps(90) + ifb.riapi_flip_steps(True, False)
    host = np.random.default_rng(50).integers(0, 256, (1080, 1920, 4), dtype=np.uint8)
    src = torch.from_numpy(host).cuda()
    before = b.kernel_launches
    out = b.orient([ifb.apply_orientation(ifb.BitmapWindow.from_torch(src), ifb.orientation_of(steps))], stream="own")[0]
    b.sync()
    assert b.kernel_launches == before + 1
    want = oo.run_nodes(host, [("ApplyOrientation", 6), oo.ROTATE_90, oo.FLIP_H])
    assert np.array_equal(out._keep.cpu().numpy(), want)


def test_flag_6_then_the_config_2_resample_equals_the_oracle():
    """a 3840x2160 frame with EXIF orientation 6 (a portrait phone photo), then 2160x3840 -> 288x512 Robidoux in linear light: the
    one-call orientation followed by the device resample against the oracle's FlipV + transpose followed by its scale_and_render"""
    import torch
    ifb = _ifb()
    b = ifb.Batch(0)
    inp = oracle.synth_noise(3840, 2160, seed=11, alpha_mode="mixed")
    mid = oo.run_nodes(inp, [("ApplyOrientation", 6)])
    want = np.zeros((512, 288, 4), np.uint8)
    oracle.scale_and_render(mid, want, filter=2, linear=True, alpha_meaningful=True)
    src = torch.from_numpy(inp).cuda()
    rot = b.orient([ifb.apply_orientation(ifb.BitmapWindow.from_torch(src, alpha_meaningful=True), 6)], stream="own")[0]
    out = torch.zeros((512, 288, 4), dtype=torch.uint8, device="cuda")
    b.scale_and_render_many([(rot, ifb.BitmapWindow.from_torch(out), ifb.ScaleAndRenderParams(w=288, h=512))], stream="own")
    b.sync()
    assert np.array_equal(rot._keep.cpu().numpy(), mid)
    got = out.cpu().numpy()
    assert np.array_equal(got, want), np.argwhere(np.any(got != want, axis=2))[:4].tolist()
