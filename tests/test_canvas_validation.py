"""Argument checks of ifb200_batch_canvas, which come before any device use: the product's own checks (ifb_canvas.cc) through the
CPU emulation of the call (tests/cpu_emu/canvas_kernel_emu.cc), where a rejected call must also write nothing; the library's null
batch and array answers; and the checks the Python mirror makes as the reference's callers do.  No GPU is needed."""
import ctypes as C

import numpy as np
import pytest

import imageflow_b200 as ifb
from imageflow_b200._lib import CanvasDesc
from tests import cpu_emu
from tests.cpu_emu import run_canvas_cases as rcc

FILL, COPY, EXPAND, NORMALIZE = range(4)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return rcc.load(cpu_emu.build(str(tmp_path_factory.mktemp("canvas_emu")), *rcc.SOURCES))


def _call(L, descs):
    arr = (CanvasDesc * len(descs))(*descs)
    cap = 1 << 12
    loads, stores = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    nl, ns = C.c_size_t(), C.c_size_t()
    err = C.create_string_buffer(256)
    ctas = L.emu_canvas(arr, len(descs), loads.ctypes.data, stores.ctypes.data, cap, C.byref(nl), C.byref(ns), err, 256, 0)
    return ctas, ns.value, err.value.decode()


def _d(op, px=None, w=8, h=6, stride=32, am=0, inp=None, in_w=8, in_h=6, in_stride=32, in_am=0, r=(0, 0, 0, 0), cw=0, ch=0, color=(1, 2, 3, 4)):
    d = CanvasDesc()
    d.op = op; d.px = px; d.w = w; d.h = h; d.stride = stride; d.alpha_meaningful = am
    d.in_ = inp; d.in_w = in_w; d.in_h = in_h; d.in_stride = in_stride; d.in_alpha_meaningful = in_am
    d.x1, d.y1, d.x2, d.y2 = r
    d.cw, d.ch = cw, ch
    d.color_bgra = (C.c_uint8 * 4)(*color)
    return d


def test_each_bad_descriptor_is_rejected_and_nothing_is_written(emu):
    cv = np.full(64 * 64 * 4, 0x5A, np.uint8)
    src = np.full(64 * 64 * 4, 0xA5, np.uint8)
    p, q = cv.ctypes.data, src.ctypes.data
    good = [_d(FILL, p, r=(0, 0, 8, 6)), _d(NORMALIZE, p + 4096), _d(COPY, p + 8192, inp=q, r=(0, 0, 1, 1), cw=4, ch=4),
            _d(EXPAND, p + 12288, w=10, h=9, stride=40, inp=q + 4096, in_w=8, in_h=6, r=(1, 2, 1, 1))]
    bad = {
        "unknown op": _d(4, p), "negative op": _d(-1, p),
        "null canvas": _d(FILL, None, r=(0, 0, 1, 1)), "null input": _d(COPY, p, inp=None, cw=1, ch=1),
        "null input of expand": _d(EXPAND, p, w=8, h=6, inp=None),
        "stride below w*4": _d(NORMALIZE, p, stride=28), "stride not a multiple of 4": _d(NORMALIZE, p, stride=34),
        "input stride below w*4": _d(COPY, p, inp=q, in_stride=20, cw=1, ch=1), "misaligned pointer": _d(NORMALIZE, p + 2),
        "fill x2 beyond w": _d(FILL, p, r=(0, 0, 9, 1)), "fill y2 beyond h": _d(FILL, p, r=(0, 0, 1, 7)),
        "fill x2 < x1": _d(FILL, p, r=(3, 0, 2, 1)), "fill y2 < y1": _d(FILL, p, r=(0, 3, 1, 2)),
        "copy from_x at in_w": _d(COPY, p, inp=q, r=(8, 0, 0, 0), cw=0, ch=1),
        "copy beyond input": _d(COPY, p, inp=q, r=(5, 0, 0, 0), cw=4, ch=1),
        "copy beyond canvas": _d(COPY, p, inp=q, r=(0, 0, 6, 4), cw=3, ch=3),
        "copy from_x + w wraps": _d(COPY, p, inp=q, r=(1, 0, 0, 0), cw=0xFFFFFFFF, ch=1),
        "copy to_y + h wraps": _d(COPY, p, inp=q, r=(0, 0, 0, 2), cw=1, ch=0xFFFFFFFE),
        "zero-width copy": _d(COPY, p, inp=q, cw=0, ch=2), "zero-height copy": _d(COPY, p, inp=q, cw=2, ch=0),
        "overlapping input and canvas": _d(COPY, p, inp=p + 32 * 5, cw=1, ch=1),
        "input inside the canvas's stride padding span": _d(COPY, p, w=4, stride=64, inp=p + 16, in_w=4, in_stride=64, cw=1, ch=1),
        "expand width mismatch": _d(EXPAND, p, w=11, h=9, stride=44, inp=q, r=(1, 2, 1, 1)),
        "expand height mismatch": _d(EXPAND, p, w=10, h=8, stride=40, inp=q, r=(1, 2, 1, 1)),
        "expand sizes wrap": _d(EXPAND, p, w=7, h=6, stride=28, inp=q, r=(0xFFFFFFFF, 0, 0, 0)),
        "expand of an empty input": _d(EXPAND, p, w=2, h=6, stride=8, inp=q, in_w=0, r=(1, 0, 1, 0)),
    }
    ok = _call(emu, good)
    assert ok[0] > 0 and ok[2] == ""
    for name, d in bad.items():
        before = (cv.copy(), src.copy())
        ctas, stores, err = _call(emu, good[:2] + [d] + good[2:])
        assert ctas == -1 and stores == 0 and "canvas job 2" in err, (name, ctas, err)
        assert np.array_equal(cv, before[0]) and np.array_equal(src, before[1]), name


def test_zero_size_fill_is_a_no_op_anywhere(emu):
    cv = np.zeros(8 * 6 * 4, np.uint8)
    for r in [(3, 2, 3, 9), (50, 60, 70, 60), (0, 0, 0, 0), (100, 1, 100, 0)]:
        ctas, stores, err = _call(emu, [_d(FILL, cv.ctypes.data, r=r)])
        assert (ctas, stores, err) == (0, 0, ""), r
    assert (cv == 0).all()


def test_null_batch_or_array_is_an_argument_error():
    buf = C.create_string_buffer(256)
    L = ifb.lib()
    assert L.ifb200_batch_canvas(None, None, 0, None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)
    assert L.ifb200_batch_canvas(None, (CanvasDesc * 1)(), 1, None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)


def test_python_mirror_checks_what_the_reference_callers_check():
    if ifb.device_count() > 0:
        pytest.skip("a CUDA device is present: tests/test_canvas_gpu.py covers Batch.canvas")
    win = ifb.BitmapWindow.from_numpy(np.zeros((6, 8, 4), np.uint8))
    # Batch needs a device; the checks run before it is used, in the op records' own marshalling
    from imageflow_b200.graphics import _fill_canvas_desc
    with pytest.raises(ifb.FlowError) as e:
        _fill_canvas_desc(CanvasDesc(), ifb.EnableTransparency(ifb.BitmapWindow.from_numpy(np.zeros((2, 2, 4), np.uint8), alpha_meaningful=True)), 0)
    assert e.value.kind == ifb.ErrorKind.InvalidArgument
    matte = ifb.BitmapWindow.from_numpy(np.zeros((6, 8, 4), np.uint8), compose=ifb.BitmapCompositing.BlendWithMatte)
    with pytest.raises(ifb.FlowError):
        _fill_canvas_desc(CanvasDesc(), ifb.FillRect(matte, 0, 0, 4, 4, (0, 0, 0, 255)), 0)
    _fill_canvas_desc(CanvasDesc(), ifb.FillRect(matte, 0, 0, 8, 6, (0, 0, 0, 255)), 0)      # the whole bitmap is allowed
    with pytest.raises(ifb.FlowError):
        _fill_canvas_desc(CanvasDesc(), ifb.FillRect(ifb.BitmapWindow.from_numpy(np.zeros((2, 2, 4), np.uint8), pixel_layout="BGR"), 0, 0, 1, 1, (0, 0, 0, 0)), 0)
    assert win.alpha_meaningful is False


def test_red_dot_and_region_helpers():
    win = ifb.BitmapWindow.from_numpy(np.zeros((3, 3, 4), np.uint8))
    assert ifb.watermark_red_dot(win) == []
    win4 = ifb.BitmapWindow.from_numpy(np.zeros((4, 5, 4), np.uint8))
    (op,) = ifb.watermark_red_dot(win4)
    assert (op.x1, op.y1, op.x2, op.y2, tuple(op.color)) == (2, 1, 5, 4, (0, 0, 255, 255))
    big = ifb.BitmapWindow.from_numpy(np.zeros((200, 200, 4), np.uint8), alpha_meaningful=True)
    e = ifb.region(big, -10, -10, 120, 50, (0, 0, 0, 0))
    assert isinstance(e, ifb.ExpandCanvas) and (e.left, e.top, e.right, e.bottom) == (10, 10, 0, 0)
    assert (e.input.w, e.input.h, e.input.ptr) == (120, 50, big.ptr)
    e = ifb.region_percent(big, -10, -10, 40, 40, (0, 0, 0, 0))
    assert (e.left, e.top, e.input.w, e.input.h) == (20, 20, 80, 80)
    with pytest.raises(ifb.FlowError):
        ifb.region(big, 5, 5, 5, 9, (0, 0, 0, 0))
