"""Argument checks and planning of ifb200_batch_color_chain, which come before any device use: the product's own checks and planner
(ifb_color.cc) through the CPU emulation of the call (tests/cpu_emu/color_kernel_emu.cc), where a rejected call must also write
nothing; the table fold against the step-by-step oracle; the segments a chain compiles into; the size of the plan, which grows with
jobs and steps and not with pixels; the library's null batch and array answers; and the Python mirror's own checks.  No GPU is
needed."""
import ctypes as C

import numpy as np
import pytest

import imageflow_b200 as ifb
from imageflow_b200._lib import ColorDesc
from tests import color_oracle as co
from tests import cpu_emu
from tests.cpu_emu import run_color_cases as rcc

TABLE, MATRIX, WB = 0, 1, 2


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return rcc.load(cpu_emu.build(str(tmp_path_factory.mktemp("color_emu")), *rcc.SOURCES))


def _call(L, descs):
    arr = (ColorDesc * max(len(descs), 1))(*descs)
    cap = 1 << 14
    loads, stores, hist = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    nl, ns, nwb, nla = C.c_size_t(), C.c_size_t(), C.c_size_t(), C.c_int()
    err = C.create_string_buffer(256)
    ctas = L.emu_color(arr, len(descs), loads.ctypes.data, stores.ctypes.data, cap, C.byref(nl), C.byref(ns), hist.ctypes.data, cap,
                       C.byref(nwb), C.byref(nla), err, 256, 0)
    return ctas, ns.value, nla.value, err.value.decode()


def _plan(L, descs):
    arr = (ColorDesc * max(len(descs), 1))(*descs)
    nb, nj, nsg = C.c_size_t(), C.c_size_t(), C.c_size_t()
    kinds = np.zeros(256, np.uint32)
    ctas = L.emu_color_plan(arr, len(descs), C.byref(nb), C.byref(nj), kinds.ctypes.data, 256, C.byref(nsg))
    return ctas, nb.value, nj.value, kinds[:nsg.value].tolist()


def _tables(L, d):
    out = np.zeros(1 << 16, np.uint8)
    n = L.emu_color_tables((ColorDesc * 1)(d), 1, out.ctypes.data, out.size)
    return out[:n].reshape(-1, 4, 256)


KEEP = []


def _d(ptr, w, h, stride, chain, am=1, n_steps=None):
    d = rcc.desc(ptr, w, h, stride, am, chain, KEEP)
    if n_steps is not None:
        d.n_steps = n_steps
    return d


def test_each_bad_descriptor_is_rejected_and_nothing_is_written(emu):
    buf = np.full(64 * 64 * 4, 0xA5, np.uint8)
    p = buf.ctypes.data
    ch = co.preset(co.BRIGHTNESS, 0.2)
    good = [_d(p, 8, 6, 32, ch), _d(p + 4096, 8, 6, 32, ch + [("white_balance", None)]), _d(p + 8192, 5, 3, 20, co.preset(co.SEPIA))]
    nan_wb = [("white_balance", float("nan"))]
    unknown = rcc.steps_array(ch); unknown[0].kind = 7; KEEP.append(unknown)
    bad_kind = _d(p, 8, 6, 32, ch); bad_kind.steps = C.cast(unknown, C.c_void_p).value
    null_steps = _d(p, 8, 6, 32, ch); null_steps.steps = None
    bad = {"null bitmap": (_d(None, 8, 6, 32, ch), 1), "null steps": (null_steps, 1), "stride below a row": (_d(p, 8, 6, 28, ch), 1),
           "stride not a multiple of 4": (_d(p, 8, 6, 34, ch), 1), "misaligned bitmap": (_d(p + 2, 8, 6, 32, ch), 1),
           "unknown step kind": (bad_kind, 1), "NaN threshold": (_d(p, 8, 6, 32, nan_wb), 1),
           "too many steps": (_d(p, 8, 6, 32, ch * 17), 1), "window too large": (_d(p, 0x10000, 0x10001, 0x40000, ch), 1),
           "second white balance": (_d(p, 8, 6, 32, [("white_balance", None)] + ch + [("white_balance", 0.1)]), 2)}
    ok = _call(emu, good)
    assert ok[0] > 0 and ok[2] == 3 and ok[3] == ""
    for name, (d, code) in bad.items():
        buf[:] = 0xA5
        ctas, stores, launches, err = _call(emu, good[:2] + [d] + good[2:])
        assert ctas == -code and stores == 0 and launches == 0 and "color job 2" in err, (name, ctas, err)
        assert (buf == 0xA5).all(), name


def test_nothing_to_write_launches_nothing(emu):
    a = np.zeros(8 * 6 * 4, np.uint8)
    p = a.ctypes.data
    et = [("enable_transparency",)]
    for d in [_d(p, 8, 6, 32, []), _d(None, 0, 6, 0, et), _d(p + 1, 8, 0, 3, et), _d(None, 8, 6, 32, [], n_steps=0),
              _d(p, 8, 6, 32, et, am=1), _d(p, 8, 6, 32, et * 3, am=1)]:                         # EnableTransparency on Bgra32 deletes itself
        assert _call(emu, [d]) == (0, 0, 0, ""), (d.w, d.h, d.n_steps)
    assert _call(emu, []) == (0, 0, 0, "")
    assert (a == 0).all()


def _all_bytes_image():
    """256 pixels whose every channel is the pixel's index"""
    return np.repeat(np.arange(256, dtype=np.uint8)[:, None], 4, axis=1).reshape(1, 256, 4)


def _fold_matches(emu, chain, am):
    """the planner's one table for a separable chain against the oracle's node-by-node result on every byte value"""
    img = _all_bytes_image()
    t = _tables(emu, _d(img.ctypes.data, 256, 1, 1024, chain, am=am))
    assert t.shape[0] == 1
    want, _, _ = co.run_chain(img, chain, am)
    return all(np.array_equal(t[0][k], want[0, :, k]) for k in range(4))


@pytest.mark.parametrize("which", [co.INVERT, co.ALPHA, co.CONTRAST, co.BRIGHTNESS])
def test_table_fold_equals_the_step_by_step_oracle_for_separable_presets(emu, which):
    for p in np.linspace(-2.0, 2.0, 41, dtype=np.float32):
        for am in (0, 1):
            assert _fold_matches(emu, co.preset(which, float(p)), am), (which, p, am)
    ps = [-0.3, 0.25, 0.7]
    chain = [s for p in ps for w in (co.BRIGHTNESS, co.CONTRAST, co.ALPHA, co.INVERT) for s in co.preset(w, p)]
    assert _fold_matches(emu, chain[:16], 0)


def test_table_fold_for_random_sparse_matrices_with_signed_zeros(emu):
    rng = np.random.default_rng(7)
    n = 0
    while n < 300:
        m = rcc.sparse_matrix(rng)
        if any(m[k, c] != 0 for k in range(4) for c in range(4) if k != c):
            continue
        chain = [("matrix", m)]
        with np.errstate(invalid="ignore", over="ignore"):
            assert _fold_matches(emu, chain, 1), m
        n += 1


def test_chains_split_into_table_matrix_table(emu):
    p = 1 << 20                                                # never dereferenced: only planned
    b, s, c = co.preset(co.BRIGHTNESS, 0.1), co.preset(co.SEPIA), co.preset(co.CONTRAST, 0.2)
    assert _plan(emu, [_d(p, 64, 64, 256, b + s + c)])[3] == [TABLE, MATRIX, TABLE]
    assert _plan(emu, [_d(p, 64, 64, 256, b + c + co.preset(co.INVERT))])[3] == [TABLE]
    assert _plan(emu, [_d(p, 64, 64, 256, co.preset(co.SATURATION, -0.5) + s)])[3] == [MATRIX, MATRIX]
    assert _plan(emu, [_d(p, 64, 64, 256, co.preset(co.ALPHA, 0.5), am=0)])[3] == [TABLE]
    assert _plan(emu, [_d(p, 64, 64, 256, b + [("white_balance", None)] + c)])[3] == [TABLE, WB, TABLE]
    assert _plan(emu, [_d(p, 64, 64, 256, co.riapi_steps(**{"alpha": 0.5, "brightness": 0.1, "contrast": 0.2, "saturation": -0.3,
                                                            "sepia": True, "grayscale": "flat", "balance_white": True}), am=0)])[3] == \
        [TABLE, MATRIX, MATRIX, MATRIX, WB]


def test_an_8k_job_with_six_steps_plans_to_a_bounded_number_of_bytes(emu):
    """what is planned and uploaded grows with jobs and steps, not pixels"""
    p = 1 << 20
    chain = co.riapi_steps(brightness=0.1, contrast=0.2, saturation=-0.3, sepia=True, grayscale="ntsc", balance_white=True)
    assert len(chain) == 6
    ctas, nbytes, nj, kinds = _plan(emu, [_d(p, 7680, 4320, 7680 * 4, chain)])
    assert nj == 1 and ctas > 1000 and nbytes <= 8192, nbytes
    ctas64, nbytes64, nj64, _ = _plan(emu, [_d(p + i * (1 << 28), 7680, 4320, 7680 * 4, chain) for i in range(64)])
    assert nj64 == 64 and ctas64 == 64 * ctas and nbytes64 <= 64 * nbytes


def test_null_batch_or_array_is_an_argument_error():
    buf = C.create_string_buffer(256)
    L = ifb.lib()
    assert L.ifb200_batch_color_chain(None, None, 0, None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)
    assert L.ifb200_batch_color_chain(None, (ColorDesc * 1)(), 1, None, buf, 256) == int(ifb.ErrorKind.InvalidArgument)


def test_python_mirror_checks_before_the_call():
    class NoBatch(ifb.Batch):                                  # the checks come before the library is called
        def __init__(self):
            self._h = C.c_void_p(); self._keep = []; self.device = 0
    b = NoBatch()
    win = ifb.BitmapWindow.from_numpy(np.zeros((6, 8, 4), np.uint8))
    for job in [(win, ["Sepia"]), (win, [ifb.EnableTransparency(win)]),
                (ifb.BitmapWindow.from_numpy(np.zeros((6, 8, 4), np.uint8), pixel_layout="BGR"), ifb.ColorFilterSrgb.sepia())]:
        with pytest.raises(ifb.FlowError) as e:
            b.color_chain([job])
        assert e.value.kind == ifb.ErrorKind.InvalidArgument
    with pytest.raises(ifb.FlowError):
        b.canvas([ifb.EnableTransparency()])
