"""Argument checks of ifb200_batch_pixel_convert, which come before any device use: the product's own checks (ifb_pixel_convert.cc)
through the CPU emulation of the call (tests/cpu_emu/pixel_convert_kernel_emu.cc), where a rejected call must also write nothing; the
size of the plan, which grows with jobs and not with pixels; the library's null batch and array answers; the Python mirror's own
checks; and the oracle against hand-derived answers.  No GPU is needed."""
import ctypes as C

import numpy as np
import pytest

import imageflow_b200 as ifb
from imageflow_b200._lib import PixelConvertDesc
from tests import cpu_emu
from tests import pixel_convert_oracle as po
from tests.cpu_emu import run_pixel_convert_cases as rpc

RGB, RGBA, GRAY, GA, TO_RGB = po.OPS


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return rpc.load(cpu_emu.build(str(tmp_path_factory.mktemp("pixel_convert_emu")), *rpc.SOURCES))


def _call(L, descs):
    arr = (PixelConvertDesc * len(descs))(*descs)
    cap = 1 << 16
    loads, stores = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    nl, ns, ni = C.c_size_t(), C.c_size_t(), C.c_size_t()
    err = C.create_string_buffer(256)
    ctas = L.emu_pixel_convert(arr, len(descs), loads.ctypes.data, stores.ctypes.data, cap, C.byref(nl), C.byref(ns), C.byref(ni),
                               err, 256, 0)
    return ctas, ns.value, err.value.decode()


def _d(op, src, src_stride, dst, dst_stride, w, h, opaque=0):
    d = PixelConvertDesc()
    d.op = op; d.src = src; d.src_stride = src_stride; d.dst = dst; d.dst_stride = dst_stride; d.w = w; d.h = h; d.opaque = opaque
    return d


def test_each_bad_descriptor_is_rejected_and_nothing_is_written(emu):
    src = np.full(1 << 16, 0xA5, np.uint8)
    dst = np.full(1 << 16, 0x5A, np.uint8)
    p, q = src.ctypes.data, dst.ctypes.data
    good = [_d(RGB, p + 1, 25, q, 32, 8, 6), _d(RGBA, p + 4096, 32, p + 4096, 32, 8, 6, 1), _d(GRAY, p + 8193, 9, q + 4096, 36, 8, 6),
            _d(TO_RGB, p + 12290, 33, q + 8195, 25, 8, 6)]
    bad = {
        "unknown op 5": _d(5, p, 32, q, 32, 8, 6), "unknown op -1": _d(-1, p, 32, q, 32, 8, 6),
        "null source pointer": _d(RGB, None, 24, q, 32, 8, 6), "null destination pointer": _d(RGB, p, 24, None, 32, 8, 6),
        "source stride smaller than a row": _d(RGB, p, 23, q, 32, 8, 6), "gray source stride": _d(GRAY, p, 7, q, 32, 8, 6),
        "gray-alpha source stride": _d(GA, p, 15, q, 32, 8, 6), "BGRA source stride": _d(TO_RGB, p, 31, q, 24, 8, 6),
        "destination stride smaller than a row": _d(RGB, p, 24, q, 28, 8, 6), "RGB destination stride": _d(TO_RGB, p, 32, q, 23, 8, 6),
        "misaligned BGRA destination": _d(RGB, p, 24, q + 2, 32, 8, 6), "BGRA destination stride not a multiple of 4": _d(GRAY, p, 8, q, 34, 8, 6),
        "misaligned in-place window": _d(RGBA, p + 1, 32, p + 1, 32, 8, 6),
        "in place with a different stride": _d(RGBA, p, 32, p, 36, 8, 6),
        "RGB24 in place": _d(RGB, p, 32, p, 32, 8, 6), "BGRA to RGB24 in place": _d(TO_RGB, p, 32, p, 32, 8, 6),
        "overlapping spans": _d(RGBA, p, 32, p + 32 * 5, 32, 8, 6),
        "destination inside the source's stride padding span": _d(GRAY, p, 64, p + 16, 64, 4, 6),
        "source starting inside the destination's last row": _d(TO_RGB, p + 5 * 64 + 3, 32, p, 64, 8, 6),
        "window too large": _d(GRAY, p, 0x40000, q, 0x40000, 0x10000, 0x10001),
    }
    ok = _call(emu, good)
    assert ok[0] > 0 and ok[2] == ""
    for name, d in bad.items():
        src[:] = 0xA5; dst[:] = 0x5A
        ctas, stores, err = _call(emu, good[:2] + [d] + good[2:])
        assert ctas == -1 and stores == 0 and err.startswith("pixel convert job 2: "), (name, ctas, err)
        assert (src == 0xA5).all() and (dst == 0x5A).all(), name


def test_messages_name_the_cause(emu):
    p = 1 << 20
    assert _call(emu, [_d(7, p, 32, p + 4096, 32, 8, 6)])[2] == "pixel convert job 0: unknown op 7"
    assert "in place with a different destination stride" in _call(emu, [_d(RGBA, p, 32, p, 64, 8, 6)])[2]
    assert "RGB24_TO_BGRA cannot run in place" in _call(emu, [_d(RGB, p, 32, p, 32, 8, 6)])[2]
    assert "4-byte aligned" in _call(emu, [_d(GA, p, 16, p + 4099, 32, 8, 6)])[2]
    assert "overlap" in _call(emu, [_d(RGBA, p, 32, p + 4, 32, 8, 6)])[2]


def test_zero_area_jobs_are_skipped_unchecked(emu):
    a = np.zeros(64, np.uint8)
    p = a.ctypes.data
    for d in [_d(RGB, None, 0, None, 0, 0, 6), _d(9, p, 0, p + 1, 0, 8, 0), _d(RGB, p, 0, p, 0, 0, 0), _d(TO_RGB, p + 1, 1, p + 3, 1, 0, 5)]:
        assert _call(emu, [d]) == (0, 0, ""), (d.op, d.w, d.h)
    assert _call(emu, []) == (0, 0, "")
    assert (a == 0).all()


@pytest.mark.parametrize("op", po.OPS)
def test_an_8k_job_plans_to_one_item(emu, op):
    """The planner's work grows with jobs, not pixels: one 7680x4320 job is one item (the launch's CTAs come from a prefix sum over
    the items), and 64 of them are 64 items and 64 times as many CTAs."""
    cs, cd = po.CHANNELS[op]
    p, q = 1 << 20, 1 << 40                                  # never dereferenced: only planned
    d = _d(op, p, 7680 * cs, q, 7680 * cd, 7680, 4320)
    ni = C.c_size_t()
    ctas = emu.emu_pixel_convert_plan((PixelConvertDesc * 1)(d), 1, C.byref(ni))
    assert ni.value == 1 and ctas == -(-(7680 * cd // 16) * 4320 // 4096)
    n64 = C.c_size_t()
    arr = (PixelConvertDesc * 64)(*[_d(op, p + i * (1 << 28), d.src_stride, q + i * (1 << 28), d.dst_stride, 7680, 4320) for i in range(64)])
    assert emu.emu_pixel_convert_plan(arr, 64, C.byref(n64)) == 64 * ctas and n64.value == 64


def test_null_batch_or_array_is_an_argument_error():
    buf = C.create_string_buffer(256)
    L = ifb.lib()
    assert L.ifb200_batch_pixel_convert(None, None, 0, None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)
    assert L.ifb200_batch_pixel_convert(None, (PixelConvertDesc * 1)(), 1, None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)


def test_python_mirror_checks_channels_and_sizes_before_the_call():
    class NoBatch(ifb.Batch):                                # the checks come before the library is called
        def __init__(self):
            self._h = C.c_void_p(); self._keep = []; self.device = 0
    b = NoBatch()
    rgb, bgra = np.zeros((6, 8, 3), np.uint8), ifb.BitmapWindow.from_numpy(np.zeros((6, 8, 4), np.uint8))
    for job in [ifb.RgbToBgra(np.zeros((6, 8, 4), np.uint8), bgra), ifb.RgbToBgra(rgb, np.zeros((6, 8, 3), np.uint8)),
                ifb.RgbToBgra(rgb, ifb.BitmapWindow.from_numpy(np.zeros((6, 7, 4), np.uint8))), ifb.BgraToRgb(bgra, np.zeros((6, 8, 4), np.uint8)),
                ifb.GrayToBgra(np.zeros((6, 8, 2), np.uint8), bgra), ifb.GrayAlphaToBgra(np.zeros((6, 8, 1), np.uint8), bgra)]:
        with pytest.raises(ifb.FlowError) as e:
            b.pixel_convert([job])
        assert e.value.kind == ifb.ErrorKind.InvalidArgument and "channel rows" in str(e.value)
    for bad in [np.zeros((6, 8, 5), np.uint8), np.zeros((6, 8), np.uint8), np.zeros((6, 8, 3), np.uint16), np.zeros((6, 8, 3), np.uint8)[:, ::-1],
                np.zeros((3, 6, 8), np.uint8).transpose(1, 2, 0)]:
        with pytest.raises(ifb.FlowError):
            ifb.PixelRows.of(bad)
    with pytest.raises(ifb.FlowError):
        b.pixel_convert([(rgb, bgra)])


def test_python_row_views_take_any_row_stride_and_byte_offset():
    a = np.zeros((10, 64), np.uint8)
    r = ifb.PixelRows.of(a[2:7, 3:3 + 3 * 9].reshape(5, 9, 3))
    assert (r.w, r.h, r.stride, r.channels, r.ptr - a.ctypes.data) == (9, 5, 64, 3, 2 * 64 + 3)
    w = ifb.PixelRows.of(ifb.BitmapWindow.from_numpy(np.zeros((4, 5, 4), np.uint8)))
    assert (w.w, w.h, w.stride, w.channels) == (5, 4, 20, 4)
    assert ifb.pixel_op_for(3) is ifb.RgbToBgra and ifb.pixel_op_for(3, to_bgra=False) is ifb.BgraToRgb
    assert ifb.pixel_op_for(1) is ifb.GrayToBgra and ifb.pixel_op_for(2) is ifb.GrayAlphaToBgra and ifb.pixel_op_for(4) is ifb.RgbaToBgra
    with pytest.raises(ifb.FlowError):
        ifb.pixel_op_for(1, to_bgra=False)


# ---------------------------------------------------------------------------------------------- the oracle, by hand
def test_oracle_matches_hand_derived_answers():
    rgb = np.array([[[10, 20, 30], [1, 2, 3]]], np.uint8)
    assert po.convert(RGB, rgb).tolist() == [[[30, 20, 10, 255], [3, 2, 1, 255]]]
    rgba = np.array([[[10, 20, 30, 40], [5, 6, 7, 0]]], np.uint8)
    assert po.convert(RGBA, rgba).tolist() == [[[30, 20, 10, 40], [7, 6, 5, 0]]]
    assert po.convert(RGBA, rgba, opaque=True).tolist() == [[[30, 20, 10, 255], [7, 6, 5, 255]]]
    assert po.convert(GRAY, np.array([[[0], [77]]], np.uint8)).tolist() == [[[0, 0, 0, 255], [77, 77, 77, 255]]]
    assert po.convert(GA, np.array([[[9, 0], [200, 128]]], np.uint8)).tolist() == [[[9, 9, 9, 0], [200, 200, 200, 128]]]
    assert po.convert(GA, np.array([[[9, 0]]], np.uint8), opaque=True).tolist() == [[[9, 9, 9, 255]]]
    bgra = np.array([[[30, 20, 10, 0], [3, 2, 1, 255]]], np.uint8)
    assert po.convert(TO_RGB, bgra).tolist() == [[[10, 20, 30], [1, 2, 3]]]
    assert po.convert(TO_RGB, bgra, opaque=True).tolist() == [[[10, 20, 30], [1, 2, 3]]]


def test_oracle_round_trips_are_the_identity():
    rng = np.random.default_rng(4)
    rgb = rng.integers(0, 256, (7, 11, 3), dtype=np.uint8)
    rgba = rng.integers(0, 256, (7, 11, 4), dtype=np.uint8)
    assert np.array_equal(po.convert(TO_RGB, po.convert(RGB, rgb)), rgb)
    assert np.array_equal(po.convert(RGBA, po.convert(RGBA, rgba)), rgba)
