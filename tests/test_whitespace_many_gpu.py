"""ifb200_batch_detect_content_many (Batch.detect_content_many) and the CropWhitespace node (Batch.crop_whitespace) on the GPU, against
the CPU oracle and against the per-frame Batch.detect_content; the reference's trim tests (imageflow_core tests/integration/visuals/
trim.rs:54-157) as device chains, bit-exact against the oracle's chain."""
import numpy as np
import pytest

import oracle
from tests.test_whitespace_product import _images

pytestmark = pytest.mark.gpu


def _dev(a, am):
    """a (h, w, 4) uint8 array in a device bitmap with rows padded to 64 bytes -> (tensor, BitmapWindow)"""
    import torch
    import imageflow_b200 as ifb
    h, w = a.shape[:2]
    pitch = (w * 4 + 63) // 64 * 64
    t = torch.zeros((h, pitch), dtype=torch.uint8, device="cuda")
    v = t.as_strided((h, w, 4), (pitch, 4, 1))
    v.copy_(torch.from_numpy(np.ascontiguousarray(a)))
    return t, ifb.BitmapWindow.from_torch(v, alpha_meaningful=am)


def _product_shot(w, h, seed):
    rng = np.random.default_rng(seed)
    a = np.full((h, w, 4), 255, np.uint8)
    x1, y1 = w // 10 + int(rng.integers(0, w // 20 + 1)), h // 10 + int(rng.integers(0, h // 20 + 1))
    a[y1:h - h // 8, x1:w - w // 9] = rng.integers(0, 256, (h - h // 8 - y1, w - w // 9 - x1, 4), dtype=np.uint8)
    return a


def test_whole_corpus_in_one_call_matches_oracle_and_per_frame_calls():
    import torch
    import imageflow_b200 as ifb
    cases = list(_images(120, 23))
    cases += [(_product_shot(3840, 2160, 1), 1, True), (_product_shot(3840, 2160, 2), 40, False), (_product_shot(7680, 4320, 3), 80, True),
              (np.zeros((1, 1, 4), np.uint8), 1, True), (np.zeros((600, 800, 4), np.uint8), 0, False)]
    b = ifb.Batch(0)
    devs = [_dev(a, am) for a, _, am in cases]
    st = torch.cuda.current_stream().cuda_stream
    rects, visited = b.detect_content_many([(win, thr) for (_, win), (_, thr, _) in zip(devs, cases)], visited=True, stream=st)
    assert len(rects) == len(cases)
    for (a, thr, am), (_, win), got, n in zip(cases, devs, rects, visited):
        want, wn = oracle.detect_content(a, thr, am)
        assert got == want and n == wn, (a.shape, thr, am, got, want, n, wn)
        assert b.detect_content(win, thr, stream=st) == want, (a.shape, thr, am)
    b.close()


@pytest.mark.parametrize("n", [1, 7, 64])
def test_two_launches_whatever_the_number_of_frames(n):
    import imageflow_b200 as ifb
    b = ifb.Batch(0)
    frames = [_dev(_product_shot(int(64 + 37 * i), int(48 + 11 * i), i), i % 2 == 0) for i in range(n)]
    before = b.kernel_launches
    rects = b.detect_content_many([(win, 30) for _, win in frames])
    assert b.kernel_launches - before == 2
    assert rects[0] == oracle.detect_content(_product_shot(64, 48, 0), 30, True)[0]
    small = [_dev(np.full((h, w, 4), 9, np.uint8), True) for w, h in [(1, 1), (2, 7), (9, 2), (2, 2)]]
    before = b.kernel_launches
    assert b.detect_content_many([(win, 1) for _, win in small]) == [(0, 0, 1, 1), (0, 0, 2, 7), (0, 0, 9, 2), (0, 0, 2, 2)]
    assert b.kernel_launches == before
    b.close()


def test_bad_descriptors_write_nothing_and_launch_nothing():
    import ctypes as C
    import imageflow_b200 as ifb
    from imageflow_b200._lib import DetectContentDesc
    b = ifb.Batch(0)
    t, win = _dev(_product_shot(64, 48, 5), True)
    for fields, msg in [(dict(px=0), "null bitmap pointer"), (dict(w=0), "empty bitmap"), (dict(stride=4), "stride smaller"),
                        (dict(px=win.ptr + 2), "not 4-byte aligned"), (dict(h=0x80000000), "oversized bitmap"),
                        (dict(threshold=0x80000000), "threshold out of range")]:
        arr = (DetectContentDesc * 3)()
        for d in arr:
            d.px, d.w, d.h, d.stride, d.alpha_meaningful, d.threshold = win.ptr, win.w, win.h, win.stride, 1, 1
        for k, v in fields.items():
            setattr(arr[1], k, v)
        rects, vis = np.full((3, 4), 7, np.uint32), np.full(3, 7, np.uint64)
        buf = C.create_string_buffer(512)
        before = b.kernel_launches
        rc = ifb.lib().ifb200_batch_detect_content_many(b._h, arr, 3, rects.ctypes.data, vis.ctypes.data, b._stream(None), buf, 512)
        assert rc == int(ifb.ErrorKind.InvalidArgument) and buf.value.decode().startswith("detect_content job 1: ") and msg in buf.value.decode()
        assert b.kernel_launches == before and (rects == 7).all() and (vis == 7).all()
    b.close()


def _bgra(hexrgba):
    v = int(hexrgba, 16)
    return ((v >> 8) & 255, (v >> 16) & 255, (v >> 24) & 255, v & 255)


def _canvas_chain(b, w, h, bg, rect, color):
    """CreateCanvas + FillRect on the device through Batch.canvas, and the same canvas in numpy"""
    import imageflow_b200 as ifb
    cv = ifb.new_canvas(w, h)
    b.canvas([ifb.FillRect(cv, 0, 0, w, h, bg)])
    b.canvas([ifb.FillRect(cv, *rect, color)])
    a = np.zeros((h, w, 4), np.uint8); a[...] = bg
    a[rect[1]:rect[3], rect[0]:rect[2]] = color
    return cv, a


def _host(win):
    import torch
    t = torch.as_strided(win._keep, (win.h, win.w, 4), (win.stride, 4, 1), win.ptr - win._keep.untyped_storage().data_ptr())
    return t.cpu().numpy()


TRIMS = [  # trim.rs: (w, h, background, FillRect, colour, threshold, percent_padding, resample)
    ("blue_dot_trimmed", 200, 200, "FFFFFFFF", (80, 80, 120, 120), "0000FFFF", 80, 0.0, None),
    ("blue_dot_padded_10pct", 200, 200, "FFFFFFFF", (80, 80, 120, 120), "FF0000FF", 80, 10.0, None),
    ("green_on_transparent", 300, 300, "00000000", (100, 100, 200, 200), "00FF00FF", 1, 0.0, None),
    ("trimmed_then_300x300", 400, 400, "FFFFFFFF", (50, 50, 150, 150), "FF5500FF", 80, 0.0, (300, 300)),
]


@pytest.mark.parametrize("case", TRIMS, ids=[t[0] for t in TRIMS])
def test_reference_trim_chains_bit_exact(case):
    import torch
    import imageflow_b200 as ifb
    _, w, h, bg, rect, color, thr, pad, resample = case
    b = ifb.Batch(0)
    cv, a = _canvas_chain(b, w, h, _bgra(bg), rect, _bgra(color))
    (cropped,) = b.crop_whitespace([(cv, ifb.CropWhitespace(thr, pad))])
    want_rect = oracle.detect_content(a, thr, True)[0]
    x1, y1, x2, y2 = ifb.crop_whitespace_bounds(want_rect, w, h, pad)
    want = a[y1:y2, x1:x2]
    assert (cropped.w, cropped.h) == (x2 - x1, y2 - y1) and cropped.ptr == cv.ptr + y1 * cv.stride + x1 * 4
    torch.cuda.synchronize()
    assert np.array_equal(_host(cropped), want)
    if resample:
        rw, rh = resample
        out = ifb.new_canvas(rw, rh)
        b.scale_and_render_many([(cropped, out, ifb.ScaleAndRenderParams(w=rw, h=rh, interpolation_filter=ifb.Filter.Robidoux))])
        torch.cuda.synchronize()
        exp = np.zeros((rh, rw, 4), np.uint8)
        oracle.scale_and_render(np.ascontiguousarray(want), exp, filter=int(ifb.Filter.Robidoux), alpha_meaningful=True)
        assert np.array_equal(_host(out), exp)
    b.close()


def test_last_column_frame_raises_invalid_state_naming_its_job():
    import imageflow_b200 as ifb
    b = ifb.Batch(0)
    a = np.zeros((50, 60, 4), np.uint8); a[:, 59] = (0, 0, 255, 255)
    assert oracle.detect_content(a, 1, True)[0] == (59, 0, 59, 49)
    _, good = _dev(_product_shot(64, 48, 7), True)
    _, bad = _dev(a, True)
    assert b.detect_content_many([(good, 1), (bad, 1)])[1] == (59, 0, 59, 49)
    with pytest.raises(ifb.FlowError, match="crop_whitespace job 1: Whitespace detection returned invalid rectangle") as e:
        b.crop_whitespace([(good, ifb.CropWhitespace(1)), (bad, ifb.CropWhitespace(1))])
    assert e.value.kind == ifb.ErrorKind.InvalidState
    b.close()
