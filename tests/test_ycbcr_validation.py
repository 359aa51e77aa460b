"""Argument checks of ifb200_batch_ycbcr_to_bgra, which come before any device use: the product's own checks (ifb_ycbcr.cc) through the
CPU emulation of the call (tests/cpu_emu/ycbcr_kernel_emu.cc), where a rejected call must plan and write nothing; the size of the
plan, which grows with jobs and not with pixels; the library's null batch and array answers; and the Python mirror's own checks.  No
GPU is needed."""
import ctypes as C

import numpy as np
import pytest

import imageflow_b200 as ifb
from imageflow_b200._lib import YcbcrDesc
from tests import cpu_emu
from tests.cpu_emu import run_ycbcr_cases as ryc

S444, S422, S420 = ifb.YCBCR_444, ifb.YCBCR_422, ifb.YCBCR_420


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return ryc.load(cpu_emu.build(str(tmp_path_factory.mktemp("ycbcr_emu")), *ryc.SOURCES))


def _call(L, descs):
    arr = (YcbcrDesc * len(descs))(*descs)
    cap = 1 << 18
    loads, stores = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    nl, ns, ni = C.c_size_t(), C.c_size_t(), C.c_size_t()
    err = C.create_string_buffer(256)
    ctas = L.emu_ycbcr(arr, len(descs), loads.ctypes.data, stores.ctypes.data, cap, C.byref(nl), C.byref(ns), C.byref(ni), err, 256, 0)
    return ctas, ns.value, ni.value, err.value.decode()


def _d(s, y, ys, cb, cbs, cr, crs, dst, ds, w, h):
    d = YcbcrDesc()
    d.sampling = s; d.y = y; d.y_stride = ys; d.cb = cb; d.cb_stride = cbs; d.cr = cr; d.cr_stride = crs
    d.dst = dst; d.dst_stride = ds; d.w = w; d.h = h
    return d


def _bad_cases(p, q):
    """{why: descriptor} for an 8 x 6 frame: planes in `p`'s buffer, destination in `q`'s"""
    y, cb, cr = p, p + 4096, p + 8192
    return {
        "unknown sampling 3": _d(3, y, 8, cb, 8, cr, 8, q, 32, 8, 6),
        "unknown sampling -1": _d(-1, y, 8, cb, 8, cr, 8, q, 32, 8, 6),
        "null Y plane pointer": _d(S420, None, 8, cb, 4, cr, 4, q, 32, 8, 6),
        "null Cb plane pointer": _d(S420, y, 8, None, 4, cr, 4, q, 32, 8, 6),
        "null Cr plane pointer": _d(S420, y, 8, cb, 4, None, 4, q, 32, 8, 6),
        "null destination pointer": _d(S420, y, 8, cb, 4, cr, 4, None, 32, 8, 6),
        "Y stride 7 smaller than its plane's row of 8 bytes": _d(S444, y, 7, cb, 8, cr, 8, q, 32, 8, 6),
        "Cb stride 7 smaller than its plane's row of 8 bytes": _d(S444, y, 8, cb, 7, cr, 8, q, 32, 8, 6),
        "Cr stride 3 smaller than its plane's row of 4 bytes": _d(S422, y, 8, cb, 4, cr, 3, q, 32, 8, 6),
        "Cb stride 4 smaller than its plane's row of 5 bytes": _d(S420, y, 9, cb, 4, cr, 5, q, 36, 9, 6),
        "destination stride 28 smaller than a BGRA row of 32 bytes": _d(S420, y, 8, cb, 4, cr, 4, q, 28, 8, 6),
        "BGRA destination pointer or stride not 4-byte aligned": _d(S420, y, 8, cb, 4, cr, 4, q + 2, 32, 8, 6),
        "BGRA destination pointer or stride not 4-byte aligned ": _d(S420, y, 8, cb, 4, cr, 4, q, 34, 8, 6),
        "destination overlaps the Y plane": _d(S444, y, 8, cb, 8, cr, 8, y + 16, 32, 8, 6),
        "destination overlaps the Cb plane": _d(S420, y, 8, cb, 4, cr, 4, cb - 32 * 5 - 4, 32, 8, 6),
        "destination overlaps the Cr plane": _d(S422, y, 8, cb, 4, cr, 64, cr + 64 * 5, 32, 8, 6),
        "window too large": _d(S444, y, 0x10000, cb, 0x10000, cr, 0x10000, q, 0x40000, 0x10000, 0x50000),   # 16385 groups x 0x50000 rows
    }


def test_each_bad_descriptor_is_rejected_and_nothing_is_planned_or_written(emu):
    buf = np.full(1 << 16, 0xA5, np.uint8)
    out = np.full(1 << 16, 0x5A, np.uint8)
    p, q = buf.ctypes.data + 64 - buf.ctypes.data % 64, out.ctypes.data + 64 - out.ctypes.data % 64
    good = [_d(S420, p + 12288, 8, p + 12800, 4, p + 13000, 4, q + 4096, 32, 8, 6),
            _d(S444, p + 14001, 9, p + 14500, 11, p + 15003, 8, q + 8192, 36, 8, 6),
            _d(S422, p + 16000, 8, p + 16500, 4, p + 17000, 4, q + 12288, 32, 8, 6)]
    ok = _call(emu, good)
    assert ok[0] > 0 and ok[2] == 3 and ok[3] == ""
    for why, d in _bad_cases(p, q).items():
        buf[:] = 0xA5; out[:] = 0x5A
        ctas, stores, items, err = _call(emu, good[:2] + [d] + good[2:])
        assert (ctas, stores, items) == (-1, 0, 0) and err == "ycbcr job 2: " + why.strip(), (why, ctas, err)
        assert (buf == 0xA5).all() and (out == 0x5A).all(), why


def test_zero_area_jobs_are_skipped_unchecked(emu):
    a = np.zeros(64, np.uint8)
    p = a.ctypes.data
    for d in [_d(S420, None, 0, None, 0, None, 0, None, 0, 0, 6), _d(9, p, 0, p, 0, p, 0, p + 1, 0, 8, 0)]:
        assert _call(emu, [d])[:3] == (0, 0, 0)
    assert _call(emu, []) == (0, 0, 0, "")
    assert (a == 0).all()


def test_planes_next_to_the_destination_are_not_overlaps(emu):
    """a destination that starts right after a plane's last byte is accepted"""
    a = np.zeros(1 << 14, np.uint8)
    p = a.ctypes.data + 64 - a.ctypes.data % 64
    y_end = p + 5 * 8 + 8                                       # an 8 x 6 Y plane at p, pitch 8
    d = _d(S444, p, 8, p + 4096, 8, p + 8192, 8, y_end, 32, 8, 6)
    assert _call(emu, [d])[3] == ""


@pytest.mark.parametrize("s", [S444, S422, S420])
def test_an_8k_job_plans_to_one_item(emu, s):
    """The planner's work grows with jobs, not pixels: one 7680x4320 job is one item, and 64 of them are 64 items and 64 times as many
    CTAs.  At 4:2:0 a unit is a row pair, so the CTAs are half those of a one-row sampling."""
    p, q = 1 << 20, 1 << 40                                     # never dereferenced: only planned
    cw = 7680 if s == S444 else 3840
    d = _d(s, p, 7680, p + (1 << 26), cw, p + (1 << 27), cw, q, 7680 * 4, 7680, 4320)
    ni, first = C.c_size_t(), np.zeros(2, np.uint32)
    ctas = emu.emu_ycbcr_plan((YcbcrDesc * 1)(d), 1, C.byref(ni), first.ctypes.data, 2)
    bands = 2160 if s == S420 else 4320
    assert ni.value == 1 and ctas == -(-(7680 * 4 // 16) * bands // ryc.CTA_UNITS) and first.tolist() == [0, ctas]
    n64 = C.c_size_t()
    arr = (YcbcrDesc * 64)(*[_d(s, d.y + i * (1 << 30), 7680, d.cb + i * (1 << 30), cw, d.cr + i * (1 << 30), cw, q + i * (1 << 30),
                                7680 * 4, 7680, 4320) for i in range(64)])
    assert emu.emu_ycbcr_plan(arr, 64, C.byref(n64), None, 0) == 64 * ctas and n64.value == 64


def test_null_batch_or_array_is_an_argument_error():
    buf = C.create_string_buffer(256)
    L = ifb.lib()
    assert L.ifb200_batch_ycbcr_to_bgra(None, None, 0, None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)
    assert L.ifb200_batch_ycbcr_to_bgra(None, (YcbcrDesc * 1)(), 1, None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)


def test_python_mirror_checks_sampling_and_shapes_before_the_call():
    class NoBatch(ifb.Batch):                                   # the checks come before the library is called
        def __init__(self):
            self._h = C.c_void_p(); self._keep = []; self.device = 0
    b = NoBatch()
    y = np.zeros((6, 8), np.uint8)
    c420, c444 = np.zeros((3, 4), np.uint8), np.zeros((6, 8), np.uint8)
    bgra = ifb.BitmapWindow.from_numpy(np.zeros((6, 8, 4), np.uint8))
    bad = [((y, c420, c420, 3, bgra), "unknown YCbCr sampling"),
           ((y, c420, c420, S444, bgra), "chroma planes"),
           ((y, c444, c444, S420, bgra), "chroma planes"),
           ((y, c420, np.zeros((3, 5), np.uint8), S420, bgra), "chroma planes"),
           ((y, np.zeros((6, 4), np.uint8), np.zeros((6, 4), np.uint8), S420, bgra), "chroma planes"),
           ((y, c420, c420, S420, ifb.BitmapWindow.from_numpy(np.zeros((6, 7, 4), np.uint8))), "BGRA frame"),
           ((y, c420, c420, S420, np.zeros((6, 8, 3), np.uint8)), "BGRA frame"),
           ((np.zeros((6, 8, 2), np.uint8), c420, c420, S420, bgra), "one channel")]
    for job, why in bad:
        with pytest.raises(ifb.FlowError) as e:
            b.ycbcr_to_bgra([job])
        assert e.value.kind == ifb.ErrorKind.InvalidArgument and why in str(e.value), (why, str(e.value))
    # the sampling is never inferred: at 2 x 2 the 4:2:2 and 4:2:0 planes differ only in rows, at 1 x 1 not at all
    assert ifb.ycbcr_chroma_shape(S420, 1, 1) == ifb.ycbcr_chroma_shape(S422, 1, 1) == ifb.ycbcr_chroma_shape(S444, 1, 1) == (1, 1)
    assert ifb.ycbcr_chroma_shape(S420, 2, 2) == (1, 1) and ifb.ycbcr_chroma_shape(S422, 2, 2) == (2, 1)
    assert ifb.ycbcr_chroma_shape(S420, 5, 3) == (2, 3) and ifb.ycbcr_chroma_shape(S422, 5, 3) == (3, 3)
