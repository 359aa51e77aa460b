"""Argument checks of ifb200_batch_bgra_to_ycbcr, which come before any device use: the product's own checks (ifb_ycbcr_enc.cc) through
the CPU emulation of the call (tests/cpu_emu/ycbcr_enc_kernel_emu.cc), where a rejected call must plan and write nothing; the size of
the plan, which grows with jobs and not with pixels; the library's null batch and array answers; and the Python mirror's own checks.
No GPU is needed."""
import ctypes as C

import numpy as np
import pytest

import imageflow_b200 as ifb
from imageflow_b200._lib import BgraToYcbcrDesc
from tests import cpu_emu
from tests.cpu_emu import run_ycbcr_enc_cases as rye

S444, S422, S420 = ifb.YCBCR_444, ifb.YCBCR_422, ifb.YCBCR_420


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return rye.load(cpu_emu.build(str(tmp_path_factory.mktemp("ycbcr_enc_emu")), *rye.SOURCES))


def _call(L, descs):
    arr = (BgraToYcbcrDesc * len(descs))(*descs)
    t_lin, lut = rye.tables()
    cap = 1 << 18
    loads, stores = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    nl, ns, ni = C.c_size_t(), C.c_size_t(), C.c_size_t()
    err = C.create_string_buffer(256)
    ctas = L.emu_bgra_to_ycbcr(arr, len(descs), t_lin.ctypes.data, lut.ctypes.data, loads.ctypes.data, stores.ctypes.data, cap,
                               C.byref(nl), C.byref(ns), C.byref(ni), err, 256, 0)
    return ctas, ns.value, ni.value, err.value.decode()


def _d(s, src, ss, y, ys, cb, cbs, cr, crs, w, h, alpha=0):
    d = BgraToYcbcrDesc()
    d.sampling = s; d.src = src; d.src_stride = ss; d.y = y; d.y_stride = ys; d.cb = cb; d.cb_stride = cbs; d.cr = cr; d.cr_stride = crs
    d.w = w; d.h = h; d.alpha_meaningful = alpha; d.matte_bgra[:] = (255, 255, 255, 255)
    return d


def _bad_cases(p, q):
    """{why: descriptor} for an 8 x 6 frame: source in `p`'s buffer, planes in `q`'s"""
    y, cb, cr = q, q + 4096, q + 8192
    return {
        "unknown sampling 3": _d(3, p, 32, y, 8, cb, 8, cr, 8, 8, 6),
        "unknown sampling -1": _d(-1, p, 32, y, 8, cb, 8, cr, 8, 8, 6),
        "null source pointer": _d(S420, None, 32, y, 8, cb, 4, cr, 4, 8, 6),
        "null Y plane pointer": _d(S420, p, 32, None, 8, cb, 4, cr, 4, 8, 6),
        "null Cb plane pointer": _d(S420, p, 32, y, 8, None, 4, cr, 4, 8, 6),
        "null Cr plane pointer": _d(S420, p, 32, y, 8, cb, 4, None, 4, 8, 6),
        "source stride 28 smaller than a BGRA row of 32 bytes": _d(S420, p, 28, y, 8, cb, 4, cr, 4, 8, 6),
        "Y stride 7 smaller than its plane's row of 8 bytes": _d(S444, p, 32, y, 7, cb, 8, cr, 8, 8, 6),
        "Cb stride 7 smaller than its plane's row of 8 bytes": _d(S444, p, 32, y, 8, cb, 7, cr, 8, 8, 6),
        "Cr stride 3 smaller than its plane's row of 4 bytes": _d(S422, p, 32, y, 8, cb, 4, cr, 3, 8, 6),
        "Cb stride 4 smaller than its plane's row of 5 bytes": _d(S420, p, 36, y, 9, cb, 4, cr, 5, 9, 6),
        "BGRA source pointer or stride not 4-byte aligned": _d(S420, p + 2, 32, y, 8, cb, 4, cr, 4, 8, 6),
        "BGRA source pointer or stride not 4-byte aligned ": _d(S420, p, 34, y, 8, cb, 4, cr, 4, 8, 6),
        "the Y plane overlaps the source": _d(S444, p, 32, p + 16, 8, cb, 8, cr, 8, 8, 6),
        "the Cb plane overlaps the source": _d(S420, p, 32, y, 8, p + 32 * 5 + 28, 4, cr, 4, 8, 6),
        "the Cr plane overlaps the source": _d(S422, p, 32, y, 8, cb, 4, p - 4 * 5 - 2, 4, 8, 6),
        "the Cb plane overlaps the Y plane": _d(S444, p, 32, y, 8, y + 40, 8, cr, 8, 8, 6),
        "the Cr plane overlaps the Y plane": _d(S420, p, 32, y, 16, cb, 4, y + 16 * 5 + 7, 4, 8, 6),
        "the Cr plane overlaps the Cb plane": _d(S422, p, 32, y, 8, cb, 4, cb + 4 * 5 + 3, 4, 8, 6),
        "window too large": _d(S444, p, 0x40000, y, 0x10000, cb, 0x10000, cr, 0x10000, 0x10000, 0x80000),   # 8192 runs x 0x80000 rows
    }


def test_each_bad_descriptor_is_rejected_and_nothing_is_planned_or_written(emu):
    src = np.full(1 << 16, 0xA5, np.uint8)
    out = np.full(1 << 16, 0x5A, np.uint8)
    p, q = src.ctypes.data + 4096 - src.ctypes.data % 64, out.ctypes.data + 64 - out.ctypes.data % 64
    good = [_d(S420, p + 12288, 32, q + 12288, 8, q + 12800, 4, q + 13000, 4, 8, 6),
            _d(S444, p + 14000, 36, q + 14001, 9, q + 14500, 11, q + 15003, 8, 8, 6, alpha=1),
            _d(S422, p + 16000, 32, q + 16000, 8, q + 16500, 4, q + 17000, 4, 8, 6)]
    ok = _call(emu, good)
    assert ok[0] > 0 and ok[2] == 3 and ok[3] == ""
    for why, d in _bad_cases(p, q).items():
        src[:] = 0xA5; out[:] = 0x5A
        ctas, stores, items, err = _call(emu, good[:2] + [d] + good[2:])
        assert (ctas, stores, items) == (-1, 0, 0) and err == "bgra_to_ycbcr job 2: " + why.strip(), (why, ctas, err)
        assert (src == 0xA5).all() and (out == 0x5A).all(), why


def test_zero_area_jobs_are_skipped_unchecked(emu):
    a = np.zeros(64, np.uint8)
    p = a.ctypes.data
    for d in [_d(S420, None, 0, None, 0, None, 0, None, 0, 0, 6), _d(9, p + 1, 0, p, 0, p, 0, p, 0, 8, 0)]:
        assert _call(emu, [d])[:3] == (0, 0, 0)
    assert _call(emu, []) == (0, 0, 0, "")
    assert (a == 0).all()


def test_adjacent_planes_are_not_overlaps(emu):
    """planes that start right after the source's or another plane's last byte are accepted, and the call runs"""
    a = np.zeros(1 << 14, np.uint8)
    p = a.ctypes.data + 64 - a.ctypes.data % 64
    src_end = p + 5 * 32 + 32                                   # an 8 x 6 BGRA source at p, pitch 32
    y_end = src_end + 5 * 8 + 8
    cb_end = y_end + 2 * 4 + 4                                  # 4:2:0 chroma: 4 x 3
    d = _d(S420, p, 32, src_end, 8, y_end, 4, cb_end, 4, 8, 6)
    ctas, stores, items, err = _call(emu, [d])
    assert err == "" and items == 1 and stores == 8 * 6 + 2 * 4 * 3


@pytest.mark.parametrize("s", [S444, S422, S420])
def test_an_8k_job_plans_to_one_item(emu, s):
    """The planner's work grows with jobs, not pixels: one 7680x4320 job is one item, and 64 of them are 64 items and 64 times as many
    CTAs.  At 4:2:0 a unit is a row pair, so the CTAs are half those of a one-row sampling."""
    p, q = 1 << 20, 1 << 40                                     # never dereferenced: only planned
    cw = 7680 if s == S444 else 3840
    d = _d(s, p, 7680 * 4, q, 7680, q + (1 << 26), cw, q + (1 << 27), cw, 7680, 4320)
    ni, first = C.c_size_t(), np.zeros(2, np.uint32)
    ctas = emu.emu_bgra_to_ycbcr_plan((BgraToYcbcrDesc * 1)(d), 1, C.byref(ni), first.ctypes.data, 2)
    bands = 2160 if s == S420 else 4320
    assert ni.value == 1 and ctas == -(-(7680 // rye.RUN) * bands // rye.CTA_UNITS) and first.tolist() == [0, ctas]
    n64 = C.c_size_t()
    arr = (BgraToYcbcrDesc * 64)(*[_d(s, p + i * (1 << 30), 7680 * 4, q + i * (1 << 30), 7680, d.cb + i * (1 << 30), cw,
                                      d.cr + i * (1 << 30), cw, 7680, 4320) for i in range(64)])
    assert emu.emu_bgra_to_ycbcr_plan(arr, 64, C.byref(n64), None, 0) == 64 * ctas and n64.value == 64


def test_null_batch_or_array_is_an_argument_error():
    buf = C.create_string_buffer(256)
    L = ifb.lib()
    assert L.ifb200_batch_bgra_to_ycbcr(None, None, 0, None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)
    assert L.ifb200_batch_bgra_to_ycbcr(None, (BgraToYcbcrDesc * 1)(), 1, None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)


def test_python_mirror_checks_sampling_and_shapes_before_the_call():
    class NoBatch(ifb.Batch):                                   # the checks come before the library is called
        def __init__(self):
            self._h = C.c_void_p(); self._keep = []; self.device = 0
    b = NoBatch()
    src = ifb.BitmapWindow.from_numpy(np.zeros((6, 8, 4), np.uint8))
    y = np.zeros((6, 8), np.uint8)
    c420, c444 = np.zeros((3, 4), np.uint8), np.zeros((6, 8), np.uint8)
    R = ifb.BgraToYcbcr
    bad = [(R(src, 3, y, c420, c420), "unknown YCbCr sampling"),
           (R(src, S444, y, c420, c420), "chroma planes"),
           (R(src, S420, y, c444, c444), "chroma planes"),
           (R(src, S420, y, c420, np.zeros((3, 5), np.uint8)), "chroma planes"),
           (R(src, S422, y, np.zeros((3, 4), np.uint8), np.zeros((3, 4), np.uint8)), "chroma planes"),
           (R(src, S420, np.zeros((6, 7), np.uint8), c420, c420), "Y plane"),
           (R(np.zeros((6, 8, 3), np.uint8), S420, y, c420, c420), "BGRA frame"),
           (R(src, S420, np.zeros((6, 8, 2), np.uint8), c420, c420), "one channel"),
           (R(src, S420, y, c420, c420, matte_bgra=(1, 2, 3)), "matte_bgra"),
           (R(src, S420, y, c420, c420, matte_bgra=(1, 2, 3, 256)), "matte_bgra"),
           ((src, S420, y, c420, c420), "not a BgraToYcbcr record")]
    for job, why in bad:
        with pytest.raises(ifb.FlowError) as e:
            b.bgra_to_ycbcr([job])
        assert e.value.kind == ifb.ErrorKind.InvalidArgument and why in str(e.value), (why, str(e.value))
