"""The argument checks at the entries of the C ABI (include/ifb200.h), called directly.

Every batched operation rejects a null batch.  Every drop-in call on host buffers rejects a null pointer or a bad stride before it
touches the device, so the answer is InvalidArgument with or without a GPU, and the buffer is left as it was.  An empty window is
nothing to do (Ok), except for detect_content, which rejects it.  On a GPU the batched operations answer the same inputs the same
way, without a launch."""
import ctypes as C

import numpy as np
import pytest

import imageflow_b200 as ifb
from imageflow_b200._lib import LIB_PATH, RoundCornersDesc

OK, INVALID = int(ifb.ErrorKind.Ok), int(ifb.ErrorKind.InvalidArgument)
P, U, I, Z, F = C.c_void_p, C.c_uint32, C.c_int, C.c_size_t, C.c_float

# name -> argument types before the trailing (char* err, size_t cap)
SIGS = {
    "ifb200_batch_enqueue": [P, P, Z, P],
    "ifb200_batch_color_matrix": [P, P, U, U, U, P, P],
    "ifb200_batch_apply_matte": [P, P, U, U, U, P, I, P],
    "ifb200_batch_transpose": [P, P, U, U, U, P, U, P],
    "ifb200_batch_flip_vertical": [P, P, U, U, U, P],
    "ifb200_batch_flip_horizontal": [P, P, U, U, U, P],
    "ifb200_batch_white_balance": [P, P, U, U, U, F, P],
    "ifb200_batch_block_scale": [P, P, U, U, U, P, U, I, I, P],
    "ifb200_batch_round_corners": [P, P, Z, P],
    "ifb200_batch_canvas": [P, P, Z, P],
    "ifb200_batch_orient": [P, P, Z, P],
    "ifb200_batch_color_chain": [P, P, Z, P],
    "ifb200_batch_watermark": [P, P, Z, P],
    "ifb200_batch_detect_content": [P, P, U, U, U, I, U, P, P],
    "ifb200_batch_whitespace_codes": [P, P, U, U, U, I, U, P, P],
    "ifb200_color_matrix_bgra8": [P, U, U, U, P],
    "ifb200_apply_matte_bgra8": [P, U, U, U, P, I],
    "ifb200_white_balance_srgb_bgra8": [P, U, U, U, F],
    "ifb200_flip_vertical_bgra8": [P, U, U, U],
    "ifb200_flip_horizontal_bgra8": [P, U, U, U],
    "ifb200_transpose_bgra8": [P, U, U, U, P, U],
    "ifb200_block_scale_u8": [P, U, U, U, P, U, I, I],
    "ifb200_detect_content_bgra8": [P, U, U, U, I, U, P],
    "ifb200_round_corners_bgra8": [P],
}
BATCHED = [n for n in SIGS if n.startswith("ifb200_batch_")]

_L = None


def call(name, *args):
    """-> (status, message)"""
    global _L
    if _L is None:
        _L = C.CDLL(LIB_PATH)        # its own function objects: the argument types set here do not leak into imageflow_b200.lib()
        for n, sig in SIGS.items():
            getattr(_L, n).argtypes = sig + [C.c_char_p, C.c_size_t]
            getattr(_L, n).restype = C.c_int
    err = C.create_string_buffer(256)
    return getattr(_L, name)(*args, err, 256), err.value.decode()


# Arguments that are valid apart from the batch: pointers into `buf`, a 4 x 4 BGRA window (stride 16), a 2 x 2 plane of 8 x 8 blocks
def _batched_args(name, batch, buf, n_descs):
    px, stream = buf.ctypes.data, None
    return {
        "ifb200_batch_enqueue": (batch, px, n_descs, stream),
        "ifb200_batch_color_matrix": (batch, px, 4, 4, 16, px, stream),
        "ifb200_batch_apply_matte": (batch, px, 4, 4, 16, px, 1, stream),
        "ifb200_batch_transpose": (batch, px, 16, 4, 4, px + 256, 16, stream),
        "ifb200_batch_flip_vertical": (batch, px, 4, 4, 16, stream),
        "ifb200_batch_flip_horizontal": (batch, px, 4, 4, 16, stream),
        "ifb200_batch_white_balance": (batch, px, 4, 4, 16, -1.0, stream),
        "ifb200_batch_block_scale": (batch, px, 16, 2, 2, px + 512, 16, 2, 0, stream),
        "ifb200_batch_round_corners": (batch, px, n_descs, stream),
        "ifb200_batch_canvas": (batch, px, n_descs, stream),
        "ifb200_batch_orient": (batch, px, n_descs, stream),
        "ifb200_batch_color_chain": (batch, px, n_descs, stream),
        "ifb200_batch_watermark": (batch, px, n_descs, stream),
        "ifb200_batch_detect_content": (batch, px, 4, 4, 16, 1, 80, px + 512, stream),
        "ifb200_batch_whitespace_codes": (batch, px, 4, 4, 16, 1, 80, px + 512, stream),
    }[name]


@pytest.mark.parametrize("name", BATCHED)
def test_batched_entries_reject_a_null_batch(name):
    buf = np.zeros(4096, np.uint8)
    for n_descs in (0, 1):
        rc, msg = call(name, *_batched_args(name, None, buf, n_descs))
        assert rc == INVALID and "null batch" in msg, (name, rc, msg)
    assert not buf.any()


def _window(rows=6, stride=24, seed=0):
    """rows of `stride` bytes of noise (by default room for a 5 x 6 BGRA window)"""
    return np.random.default_rng(seed).integers(0, 256, (rows, stride), dtype=np.uint8)


def _rc_desc(px, w, h, stride):
    d = RoundCornersDesc()
    d.px = px; d.w = w; d.h = h; d.stride = stride; d.mode = int(ifb.RoundCornersMode.PIXELS)
    d.radius = (C.c_float * 4)(2.0, 0, 0, 0)
    d.matte_bgra = (C.c_uint8 * 4)(1, 2, 3, 4)
    return d


def _round_corners(px, w, h, stride):
    d = _rc_desc(px, w, h, stride)
    return call("ifb200_round_corners_bgra8", C.addressof(d))


# Each in-place drop-in as f(px, w, h, stride) over a BGRA window, with valid values for its other arguments
MATRIX = (C.c_float * 25)(*np.eye(5, dtype=np.float32).ravel())
MATTE = (C.c_uint8 * 4)(9, 8, 7, 255)
RECT = (C.c_uint32 * 4)()
IN_PLACE = {
    "color_matrix": lambda px, w, h, s: call("ifb200_color_matrix_bgra8", px, w, h, s, C.addressof(MATRIX)),
    "apply_matte": lambda px, w, h, s: call("ifb200_apply_matte_bgra8", px, w, h, s, C.addressof(MATTE), 1),
    "white_balance": lambda px, w, h, s: call("ifb200_white_balance_srgb_bgra8", px, w, h, s, -1.0),
    "flip_vertical": lambda px, w, h, s: call("ifb200_flip_vertical_bgra8", px, w, h, s),
    "flip_horizontal": lambda px, w, h, s: call("ifb200_flip_horizontal_bgra8", px, w, h, s),
    "detect_content": lambda px, w, h, s: call("ifb200_detect_content_bgra8", px, w, h, s, 1, 80, C.addressof(RECT)),
    "round_corners": lambda px, w, h, s: _round_corners(px, w, h, s),
    "transpose_from": lambda px, w, h, s: call("ifb200_transpose_bgra8", px, s, w, h, TRANSPOSE_TO.ctypes.data, 64),
    "transpose_to": lambda px, w, h, s: call("ifb200_transpose_bgra8", TRANSPOSE_FROM.ctypes.data, 64, h, w, px, s),
}
TRANSPOSE_FROM, TRANSPOSE_TO = np.zeros((16, 64), np.uint8), np.zeros((16, 64), np.uint8)


@pytest.mark.parametrize("op", list(IN_PLACE))
def test_drop_in_calls_reject_bad_windows_before_the_device(op):
    """A null pointer, a stride below a row and a stride that is not a multiple of 4: InvalidArgument whether or not a device is
    present (not NoDevice), and nothing written."""
    f = IN_PLACE[op]
    for w, h, stride in [(5, 6, 0), (5, 6, 16), (5, 6, 19), (5, 6, 22)]:
        a = _window()
        before = a.copy()
        rc, msg = f(a.ctypes.data, w, h, stride)
        assert rc == INVALID, (op, stride, rc, msg)
        assert np.array_equal(a, before), (op, stride)
    rc, msg = f(None, 5, 6, 24)
    assert rc == INVALID and "null" in msg, (op, rc, msg)
    assert not TRANSPOSE_FROM.any() and not TRANSPOSE_TO.any()


@pytest.mark.parametrize("op", list(IN_PLACE))
def test_drop_in_calls_on_empty_windows(op):
    """Nothing to do, whatever the stride (Ok, nothing written), except detect_content, which rejects an empty bitmap."""
    f = IN_PLACE[op]
    a = _window()
    before = a.copy()
    for w, h, stride in [(0, 6, 24), (5, 0, 24), (0, 0, 0), (0, 6, 3)]:
        rc, msg = f(a.ctypes.data, w, h, stride)
        assert rc == (INVALID if op == "detect_content" else OK), (op, w, h, stride, rc, msg)
    assert np.array_equal(a, before)


def test_drop_in_calls_reject_other_null_pointers():
    a = _window()
    before = a.copy()
    px = a.ctypes.data
    for w, h in [(5, 6), (0, 0)]:
        assert call("ifb200_color_matrix_bgra8", px, w, h, 24, None)[0] == INVALID
        assert call("ifb200_apply_matte_bgra8", px, w, h, 24, None, 1)[0] == INVALID
        assert call("ifb200_apply_matte_bgra8", px, w, h, 24, None, 0)[0] == INVALID
        assert call("ifb200_detect_content_bgra8", px, w, h, 24, 1, 80, None)[0] == INVALID
        assert call("ifb200_transpose_bgra8", px, 24, w, h, None, 64)[0] == INVALID
        assert call("ifb200_block_scale_u8", None, 64, w, h, px, 64, 2, 0)[0] == INVALID
        assert call("ifb200_block_scale_u8", px, 64, w, h, None, 64, 2, 0)[0] == INVALID
    assert call("ifb200_round_corners_bgra8", None)[0] == INVALID
    assert np.array_equal(a, before)


def test_apply_matte_without_meaningful_alpha_does_nothing():
    """blend.rs:10-13: with alpha not meaningful the call returns before looking at the window."""
    a = _window()
    before = a.copy()
    for stride in (24, 16, 22):
        assert call("ifb200_apply_matte_bgra8", a.ctypes.data, 5, 6, stride, C.addressof(MATTE), 0) == (OK, "")
    assert np.array_equal(a, before)


def test_block_scale_drop_in_checks():
    """Plane strides below a row of blocks and block sizes outside 1..7 are argument errors; an empty plane is nothing to do."""
    src, dst = _window(16, 64, seed=1), _window(16, 64, seed=2)
    before = dst.copy()
    s, d = src.ctypes.data, dst.ctypes.data
    for args in [(s, 15, 2, 2, d, 64, 2, 0), (s, 64, 2, 2, d, 3, 2, 0), (s, 64, 2, 2, d, 64, 0, 0), (s, 64, 2, 2, d, 64, 8, 0)]:
        assert call("ifb200_block_scale_u8", *args)[0] == INVALID, args
    for args in [(s, 0, 0, 2, d, 0, 2, 0), (s, 64, 2, 0, d, 64, 2, 1)]:
        assert call("ifb200_block_scale_u8", *args) == (OK, ""), args
    assert np.array_equal(dst, before)


@pytest.mark.gpu
def test_batched_operations_check_their_windows_without_a_launch():
    import torch

    out = C.c_void_p()
    L = ifb.lib()
    err = C.create_string_buffer(256)
    assert L.ifb200_batch_create(0, C.byref(out), err, 256) == OK, err.value
    b = out.value
    try:
        dev = torch.zeros(4096, dtype=torch.uint8, device="cuda")
        px = dev.data_ptr()
        m, matte, codes = C.addressof(MATRIX), C.addressof(MATTE), px + 2048
        rect = (C.c_uint32 * 4)()
        own = C.c_void_p(-1)
        window_ops = {
            "color_matrix": lambda p, w, h, s: call("ifb200_batch_color_matrix", b, p, w, h, s, m, own),
            "apply_matte": lambda p, w, h, s: call("ifb200_batch_apply_matte", b, p, w, h, s, matte, 1, own),
            "white_balance": lambda p, w, h, s: call("ifb200_batch_white_balance", b, p, w, h, s, -1.0, own),
            "flip_vertical": lambda p, w, h, s: call("ifb200_batch_flip_vertical", b, p, w, h, s, own),
            "flip_horizontal": lambda p, w, h, s: call("ifb200_batch_flip_horizontal", b, p, w, h, s, own),
            "transpose": lambda p, w, h, s: call("ifb200_batch_transpose", b, p, s, w, h, px + 1024, 64, own),
            "detect_content": lambda p, w, h, s: call("ifb200_batch_detect_content", b, p, w, h, s, 1, 80, C.addressof(rect), own),
            "whitespace_codes": lambda p, w, h, s: call("ifb200_batch_whitespace_codes", b, p, w, h, s, 1, 80, codes, own),
        }
        launches = L.ifb200_batch_kernel_launches(b)
        for op, f in window_ops.items():
            for args in [(None, 5, 6, 24), (px, 5, 6, 16), (px, 5, 6, 22)]:
                assert f(*args)[0] == INVALID, (op, args)
            empty_ok = op not in ("detect_content", "whitespace_codes")
            for args in [(px, 0, 6, 24), (px, 5, 0, 3)]:
                assert f(*args)[0] == (OK if empty_ok else INVALID), (op, args)
        for name in ("ifb200_batch_enqueue", "ifb200_batch_round_corners", "ifb200_batch_canvas", "ifb200_batch_orient",
                     "ifb200_batch_color_chain", "ifb200_batch_watermark"):
            rc, msg = call(name, b, None, 1, own)
            assert rc == INVALID and "null descriptor array" in msg, (name, rc, msg)
            assert call(name, b, None, 0, own) == (OK, ""), name
        assert L.ifb200_batch_sync(b, err, 256) == OK, err.value
        assert L.ifb200_batch_kernel_launches(b) == launches
        assert not dev.any()
    finally:
        L.ifb200_batch_destroy(b)
