"""Argument checks of ifb200_batch_watermark, which come before any device work: every bad descriptor of a call (null pointers, a
rectangle outside the frame, an empty watermark, short or unaligned strides, a pointer off a 4-byte boundary, an unknown compositing
mode or filter, a colour matrix) is rejected with its status and nothing of the call is written; zero-area jobs are skipped unchecked;
a null batch or descriptor array is refused.  Runs on the GPU: the library has no CPU path."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _setup():
    import torch
    import imageflow_b200 as ifb
    from imageflow_b200._lib import WatermarkDesc
    from imageflow_b200 import synth
    logo = torch.from_numpy(synth.cutout_np(24, 16, 1)).cuda()
    frames = [torch.from_numpy(synth.noise_np(64, 48, s)).cuda() for s in range(3)]
    arr = (WatermarkDesc * 3)()
    for d, f in zip(arr, frames):
        ifb.graphics._fill_desc(d.draw, ifb.BitmapWindow.from_torch(logo, alpha_meaningful=True), ifb.BitmapWindow.from_torch(f),
                                ifb.ScaleAndRenderParams(x=4, y=5, w=30, h=20, interpolation_filter=ifb.Filter.Ginseng))
        d.opacity = 0.5
    return ifb, logo, frames, arr


BAD = [
    ("in_", 0, 1, b"null bitmap pointer"), ("canvas", 0, 1, b"null bitmap pointer"), ("x", 40, 1, b"out of bounds"),
    ("h", 44, 1, b"out of bounds"), ("in_w", 0, 1, b"empty bitmap"), ("in_stride", 95, 1, b"stride"), ("cv_stride", 128, 1, b"stride"),
    ("compose", 3, 1, b"compositing mode"), ("filter", 0, 13, b"filter"), ("filter", 32, 13, b"filter"),
    ("color_matrix", "matrix", 1, b"colour matrix"), ("in_", "+2", 1, b"4-byte"),
]


@pytest.mark.parametrize("field, value, code, msg", BAD, ids=[f"{b[0]}={b[1]}" for b in BAD])
def test_a_bad_descriptor_rejects_the_call_and_writes_nothing(field, value, code, msg):
    import torch
    ifb, logo, frames, arr = _setup()
    before = [f.clone() for f in frames]
    m = np.eye(5, dtype=np.float32)
    if value == "matrix":
        value = m.ctypes.data
    elif value == "+2":
        value = getattr(arr[1].draw, field) + 2
    setattr(arr[1].draw, field, value)
    b = ifb.Batch(0)
    buf = C.create_string_buffer(256)
    rc = ifb.lib().ifb200_batch_watermark(b._h, arr, 3, b.STREAM_OWN, buf, 256)
    b.sync()
    assert rc == code and msg in buf.value and b"job 1" in buf.value, (rc, buf.value)
    assert b.kernel_launches == 0
    for f, g in zip(frames, before):
        assert torch.equal(f, g)


def test_zero_area_jobs_are_skipped_unchecked_and_null_arguments_refused():
    import torch
    ifb, logo, frames, arr = _setup()
    before = [f.clone() for f in frames]
    for d in arr:
        d.draw.w = 0
        d.draw.in_ = None
    b = ifb.Batch(0)
    buf = C.create_string_buffer(256)
    assert ifb.lib().ifb200_batch_watermark(b._h, arr, 3, b.STREAM_OWN, buf, 256) == 0
    b.sync()
    assert b.kernel_launches == 0 and all(torch.equal(f, g) for f, g in zip(frames, before))
    assert ifb.lib().ifb200_batch_watermark(None, arr, 3, b.STREAM_OWN, buf, 256) == 1
    assert ifb.lib().ifb200_batch_watermark(b._h, None, 3, b.STREAM_OWN, buf, 256) == 1
    assert ifb.lib().ifb200_batch_watermark(b._h, None, 0, b.STREAM_OWN, buf, 256) == 0
