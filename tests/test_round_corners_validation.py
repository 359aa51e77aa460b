"""Argument checks of the rounded-corner entry points (include/ifb200.h), which come before any device use, and the missing-device
answer of the drop-in call.  No GPU compute is called here."""
import ctypes as C

import numpy as np
import pytest

import imageflow_b200 as ifb
from imageflow_b200._lib import RoundCornersDesc

M = ifb.RoundCornersMode


def _desc(px, w, h, stride, mode=M.PIXELS, radius=(5.0, 0, 0, 0)):
    d = RoundCornersDesc()
    d.px = px; d.w = w; d.h = h; d.stride = stride; d.mode = mode
    d.radius = (C.c_float * 4)(*radius)
    return d


def _drop_in(d):
    buf = C.create_string_buffer(256)
    return ifb.lib().ifb200_round_corners_bgra8(C.byref(d), buf, 256), buf.value.decode()


def test_bad_arguments_are_rejected_before_any_device_use():
    a = np.zeros((8, 10, 4), np.uint8)
    p = a.ctypes.data
    for d in [_desc(None, 10, 8, 40), _desc(p, 10, 8, 36), _desc(p, 10, 8, 42), _desc(p, 10, 8, 40, mode=5), _desc(p, 10, 8, 40, mode=-1),
              _desc(p, 0, 8, 40, mode=7)]:
        rc, msg = _drop_in(d)
        assert rc == int(ifb.ErrorKind.InvalidArgument), (rc, msg)
    buf = C.create_string_buffer(256)
    assert ifb.lib().ifb200_round_corners_bgra8(None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)
    assert ifb.lib().ifb200_batch_round_corners(None, None, 0, None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)
    assert (a == 0).all()


def test_empty_windows_do_nothing():
    for d in [_desc(None, 0, 8, 0), _desc(None, 8, 0, 0), _desc(None, 0, 0, 0, mode=M.CIRCLE)]:
        assert _drop_in(d) == (0, "")


def test_degenerate_radii_are_not_argument_errors():
    """NaN, infinite, negative and oversized radii have the reference's meaning; only the device can be missing."""
    if ifb.device_count() > 0:
        pytest.skip("a CUDA device is present: tests/test_round_corners_gpu.py covers these radii on it")
    a = np.zeros((8, 10, 4), np.uint8)
    for r in [float("nan"), float("inf"), -float("inf"), -3.0, 1e30]:
        for mode in range(5):
            rc, msg = _drop_in(_desc(a.ctypes.data, 10, 8, 40, mode=mode, radius=(r, r, r, r)))
            assert rc == int(ifb.ErrorKind.NoDevice) and "no CPU fallback" in msg, (r, mode, rc, msg)


def test_python_mirror_reports_no_device():
    if ifb.device_count() > 0:
        pytest.skip("a CUDA device is present")
    win = ifb.BitmapWindow.from_numpy(np.zeros((6, 6, 4), np.uint8))
    with pytest.raises(ifb.FlowError) as e:
        ifb.flow_bitmap_bgra_clear_around_rounded_corners(win, M.percentage(50), (0, 0, 0, 255))
    assert e.value.kind == ifb.ErrorKind.NoDevice
    with pytest.raises(ifb.FlowError) as e:
        ifb.flow_bitmap_bgra_clear_around_rounded_corners(ifb.BitmapWindow.from_numpy(np.zeros((6, 6, 4), np.uint8), pixel_layout="BGR"),
                                                          M.circle(), (0, 0, 0, 0))
    assert e.value.kind == ifb.ErrorKind.InvalidArgument


def test_mode_constructors_follow_the_field_order():
    assert M.pixels_custom(1, 2, 3, 4) == M(M.PIXELS_CUSTOM, (1.0, 2.0, 3.0, 4.0))
    assert M.percentage_custom(1, 2, 3, 4).kind == 3 and M.circle().kind == 2 and M.pixels(3).radius[0] == 3.0 and M.percentage(9).kind == 0
