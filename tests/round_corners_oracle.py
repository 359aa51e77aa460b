"""ctypes loader of the CPU oracle of graphics/rounded_corners.rs (TEST INFRASTRUCTURE ONLY; tests/round_corners_oracle.c).

The library is compiled on first use, together with oracle/ifb_oracle.c (the transfer tables and uchar_clamp_ff it shares with the
other oracles), into a temporary directory that is removed when the process ends: the source tree is only read."""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from oracle import OracleError

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
# the flags of oracle/Makefile: no contraction, no fast math
_CFLAGS = ["-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-std=c11"]
PERCENTAGE, PIXELS, CIRCLE, PERCENTAGE_CUSTOM, PIXELS_CUSTOM = range(5)

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    out = tempfile.mkdtemp(prefix="ifb_rc_oracle_")
    atexit.register(shutil.rmtree, out, True)
    so = os.path.join(out, "libround_corners_oracle.so")
    subprocess.run(["gcc", *_CFLAGS, "-o", so, os.path.join(_HERE, "round_corners_oracle.c"), os.path.join(_ROOT, "oracle", "ifb_oracle.c"), "-lm"],
                   check=True, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    L = C.CDLL(so)
    L.rco_round_corners.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_uint8), C.c_void_p]
    L.rco_round_corners.restype = C.c_int
    L.ifo_uchar_clamp_ff.argtypes = [C.c_float]
    L.ifo_uchar_clamp_ff.restype = C.c_uint8
    _lib = L
    return L


def round_corners(px: np.ndarray, mode: int, radius=(0.0, 0.0, 0.0, 0.0), matte_bgra=(0, 0, 0, 0), w=None, want_mask: bool = False):
    """flow_bitmap_bgra_clear_around_rounded_corners, in place on px (H, W', 4) uint8 (only the first w columns are the window).
    radius: (top_left, top_right, bottom_right, bottom_left), [0] alone for Percentage / Pixels.  Returns the (h, w) uint8 mask of
    the pixels written (1: last written with the matte, 2: blended) when want_mask, else None."""
    h = px.shape[0]
    w = px.shape[1] if w is None else w
    assert px.dtype == np.uint8 and px.strides[-1] == 1 and (px.ndim == 2 or px.strides[1] == 4)
    r = (C.c_float * 4)(*[float(v) for v in (list(radius) + [0.0] * 4)[:4]])
    mm = (C.c_uint8 * 4)(*matte_bgra)
    mask = np.zeros((h, w), np.uint8) if want_mask else None
    rc = lib().rco_round_corners(px.ctypes.data, w, h, px.strides[0], int(mode), r, mm, mask.ctypes.data if want_mask else None)
    if rc:
        raise OracleError(rc)
    return mask
