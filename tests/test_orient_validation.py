"""Argument checks of ifb200_batch_orient, which come before any device use: the product's own checks (ifb_orient.cc) through the
CPU emulation of the call (tests/cpu_emu/orient_kernel_emu.cc), where a rejected call must also write nothing; the size of the plan,
which grows with jobs and not with pixels; the library's null batch and array answers; and the Python mirror's own checks.  No GPU is
needed."""
import ctypes as C

import numpy as np
import pytest

import imageflow_b200 as ifb
from imageflow_b200._lib import OrientDesc
from tests import cpu_emu
from tests.cpu_emu import run_orient_cases as roc


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return roc.load(cpu_emu.build(str(tmp_path_factory.mktemp("orient_emu")), *roc.SOURCES))


def _call(L, descs):
    arr = (OrientDesc * len(descs))(*descs)
    cap = 1 << 14
    loads, stores = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    nl, ns, bad, ni = C.c_size_t(), C.c_size_t(), C.c_long(), C.c_size_t()
    err = C.create_string_buffer(256)
    ctas = L.emu_orient(arr, len(descs), loads.ctypes.data, stores.ctypes.data, cap, C.byref(nl), C.byref(ns), C.byref(bad), C.byref(ni),
                        err, 256, 0)
    return ctas, ns.value, err.value.decode()


def _d(inp, w, h, stride, out, out_stride, o):
    d = OrientDesc()
    d.in_ = inp; d.in_w = w; d.in_h = h; d.in_stride = stride; d.out = out; d.out_stride = out_stride; d.orientation = o
    return d


def test_each_bad_descriptor_is_rejected_and_nothing_is_written(emu):
    src = np.full(64 * 64 * 4, 0xA5, np.uint8)
    dst = np.full(64 * 64 * 4, 0x5A, np.uint8)
    p, q = src.ctypes.data, dst.ctypes.data
    good = [_d(p, 8, 6, 32, q, 24, 6), _d(p + 4096, 8, 6, 32, p + 4096, 32, 3), _d(p + 8192, 8, 6, 32, q + 4096, 32, 4),
            _d(p + 12288, 5, 3, 20, q + 8192, 12, 8)]
    bad = {
        "null input": _d(None, 8, 6, 32, q, 32, 2), "null output": _d(p, 8, 6, 32, None, 32, 2),
        "input stride below a row": _d(p, 8, 6, 28, q, 32, 2), "output stride below a row": _d(p, 8, 6, 32, q, 28, 2),
        "transposed output stride below a row": _d(p, 8, 6, 32, q, 20, 5),
        "input stride not a multiple of 4": _d(p, 8, 6, 34, q, 32, 2), "output stride not a multiple of 4": _d(p, 8, 6, 32, q, 33, 2),
        "misaligned input": _d(p + 2, 8, 6, 32, q, 32, 2), "misaligned output": _d(p, 8, 6, 32, q + 1, 32, 2),
        "in-place transpose 5": _d(p, 6, 6, 32, p, 32, 5), "in-place rotate 6": _d(p, 6, 6, 32, p, 32, 6),
        "in-place 7": _d(p, 6, 6, 32, p, 32, 7), "in-place 8": _d(p, 6, 6, 32, p, 32, 8),
        "in place with another stride": _d(p, 8, 6, 32, p, 64, 2),
        "overlapping windows": _d(p, 8, 6, 32, p + 32 * 5, 32, 2),
        "output inside the input's stride padding span": _d(p, 4, 6, 64, p + 16, 64, 4),
        "transposed output overlapping the input": _d(p, 8, 6, 256, p + 64, 256, 6),
        "window too large": _d(p, 0x10000, 0x10001, 0x40000, q, 0x40000, 2),
    }
    ok = _call(emu, good)
    assert ok[0] > 0 and ok[2] == ""
    for name, d in bad.items():
        src[:] = 0xA5; dst[:] = 0x5A
        ctas, stores, err = _call(emu, good[:2] + [d] + good[2:])
        assert ctas == -1 and stores == 0 and "orient job 2" in err, (name, ctas, err)
        assert (src == 0xA5).all() and (dst == 0x5A).all(), name


def test_nothing_to_write_launches_nothing(emu):
    a = np.zeros(8 * 6 * 4, np.uint8)
    p = a.ctypes.data
    for d in [_d(p, 8, 6, 32, p, 32, 1), _d(p, 8, 6, 32, p, 32, 0), _d(p, 8, 6, 32, p, 32, 9), _d(p, 8, 6, 32, p, 32, -1),
              _d(None, 0, 6, 0, None, 0, 6), _d(None, 8, 0, 0, None, 0, 2), _d(p + 1, 0, 0, 3, None, 0, 5),
              _d(p, 1, 1, 4, p, 4, 3), _d(p, 1, 7, 4, p, 4, 2), _d(p, 7, 1, 28, p, 28, 4)]:   # 1-pixel-wide flips have no pair
        assert _call(emu, [d]) == (0, 0, ""), (d.in_w, d.in_h, d.orientation)
    assert _call(emu, []) == (0, 0, "")
    assert (a == 0).all()


@pytest.mark.parametrize("o,in_place", [(o, False) for o in range(1, 9)] + [(o, True) for o in (2, 3, 4)])
def test_an_8k_job_plans_to_a_constant_number_of_items(emu, o, in_place):
    """The planner's work grows with jobs, not pixels: one 7680x4320 job is at most two items (the launch's CTAs come from a prefix
    sum over them), and 64 of them are 64 times as many."""
    p, q = 1 << 20, 1 << 40                                  # never dereferenced: only planned
    d = _d(p, 7680, 4320, 7680 * 4, p if in_place else q, (4320 if o >= 5 else 7680) * 4, o)
    ni = C.c_size_t()
    ctas = emu.emu_orient_plan((OrientDesc * 1)(d), 1, C.byref(ni))
    assert 1 <= ni.value <= 2 and ctas > 1000
    n64 = C.c_size_t()
    arr = (OrientDesc * 64)(*[_d(p + i * (1 << 28), 7680, 4320, 7680 * 4, p + i * (1 << 28) if in_place else q + i * (1 << 28),
                                 d.out_stride, o) for i in range(64)])
    assert emu.emu_orient_plan(arr, 64, C.byref(n64)) == 64 * ctas and n64.value == 64 * ni.value


def test_null_batch_or_array_is_an_argument_error():
    buf = C.create_string_buffer(256)
    L = ifb.lib()
    assert L.ifb200_batch_orient(None, None, 0, None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)
    assert L.ifb200_batch_orient(None, (OrientDesc * 1)(), 1, None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)


def test_python_mirror_checks_output_dimensions_before_the_call():
    class NoBatch(ifb.Batch):                                # the checks come before the library is called
        def __init__(self):
            self._h = C.c_void_p(); self._keep = []; self.device = 0
    b = NoBatch()
    win = ifb.BitmapWindow.from_numpy(np.zeros((6, 8, 4), np.uint8))
    for out, o in [(ifb.BitmapWindow.from_numpy(np.zeros((6, 8, 4), np.uint8)), 6), (ifb.BitmapWindow.from_numpy(np.zeros((8, 6, 4), np.uint8)), 2),
                   (ifb.BitmapWindow.from_numpy(np.zeros((8, 6, 4), np.uint8), pixel_layout="BGR"), 5), (None, 5)]:
        with pytest.raises(ifb.FlowError) as e:
            b.orient([(win, out, o)])
        assert e.value.kind == ifb.ErrorKind.InvalidArgument and "orientation" in str(e.value)
