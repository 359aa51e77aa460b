"""The premise of tests/test_identity_resample_gpu.py, pinned on the CPU oracle: geometries whose resample returns the loaded
pixels unchanged (F == p), so that the real kernels can be run on store inputs that are known exactly.

  * Box (24) and Triangle (22) at 1:1 are one tap of weight 1.0: fmaf(1, p, +0) == p (p is never -0);
  * Box at 2:1 is (0.5, 0.5): on an image of constant 2 x 2 blocks each pass computes fmaf(0.5, p, 0.5 p) == p exactly.
Then the store epilogue alone decides the bytes, and tests/watermark_oracle.composite (its numpy restatement) on p must equal the
oracle's bytes."""
import numpy as np
import pytest

import oracle
from tests import watermark_oracle as wo

F32 = np.float32
BLOCK = 16
MATTE = (40, 200, 90, 128)


def source(nb: int = 256, block: int = BLOCK) -> np.ndarray:
    """(nb * block)^2 BGRA pixels; block (by, bx) has colour bytes (by, 255 - by, 7 by mod 256) and alpha byte bx: with nb = 256
    every (colour, alpha) byte pair of every channel"""
    c = np.arange(nb, dtype=np.int64)
    blk = np.zeros((nb, nb, 4), np.uint8)
    blk[..., 0] = c[:, None]
    blk[..., 1] = 255 - c[:, None]
    blk[..., 2] = (7 * c[:, None]) % 256
    blk[..., 3] = c[None, :]
    return np.repeat(np.repeat(blk, block, 0), block, 1)


def canvas(nb: int = 256, block: int = BLOCK, seed: int = 3) -> np.ndarray:
    """canvas of the same size: pixel (y, x) of a block has alpha byte (y mod block) * block + x mod block (every byte for block 16),
    random colour bytes"""
    n = nb * block
    cv = np.random.default_rng(seed).integers(0, 256, (n, n, 4), dtype=np.uint8)
    yy, xx = np.mgrid[0:n, 0:n]
    cv[..., 3] = ((yy % block) * block + xx % block) % 256
    return cv


def doubled(a: np.ndarray) -> np.ndarray:
    """every pixel as a constant 2 x 2 block (the input of the 2:1 Box down-scale)"""
    return np.ascontiguousarray(np.repeat(np.repeat(a, 2, 0), 2, 1))


def premultiplied(src: np.ndarray, linear: bool) -> np.ndarray:
    """p = (T[b] af, T[g] af, T[r] af, af), af = a * (1/255f): the load step of every kernel (ifb_kernels.cuh)"""
    T = oracle.byte_to_float_table(linear)
    af = src[..., 3].astype(F32) * F32(1.0 / 255.0)
    return np.stack([T[src[..., k]] * af for k in range(3)] + [af], -1).astype(F32)


def sepia_bias() -> np.ndarray:
    """sepia with a bias row: not the tile kernel's 3x3 form (the bias must be added)"""
    m = oracle.color_filter_matrix(0).astype(F32).copy()
    m[4, :3] = [0.05, -0.03, 0.02]
    return m


def matrices():
    return {"none": None, "sepia": oracle.color_filter_matrix(0).astype(F32), "sepia+bias": sepia_bias()}


@pytest.mark.parametrize("n", [1, 7, 64, 4096])
def test_identity_weights(n):
    for flt in (24, 22):                                      # Box, Triangle at 1:1: one tap of weight 1.0
        for i, (l, r, w) in enumerate(oracle.weights(flt, n, n)):
            assert (l, r) == (i, i) and w.tolist() == [1.0], (flt, i, l, r, w)
    if n % 2 == 0:                                            # Box at 2:1: (0.5, 0.5) on source pixels 2i, 2i + 1
        for i, (l, r, w) in enumerate(oracle.weights(24, n // 2, n)):
            assert (l, r) == (2 * i, 2 * i + 1) and w.tolist() == [0.5, 0.5], (i, l, r, w)


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("geometry", ["box 1:1", "triangle 1:1", "box 2:1 on 2x2 blocks"])
def test_resample_returns_the_loaded_pixels(linear, geometry):
    """oracle.resample_stages: F == p bit for bit, for every (colour, alpha) byte pair"""
    src = source(256, 1)
    p = premultiplied(src, linear)
    inp = doubled(src) if geometry.startswith("box 2:1") else src
    flt = 22 if geometry.startswith("triangle") else 24
    f = wo.f_of(inp, True, 256, 256, flt, linear=linear)
    assert np.array_equal(f.view(np.uint32), p.view(np.uint32)), geometry


@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("compose", [0, 1, 2])
def test_composite_of_p_equals_the_oracle(linear, compose):
    """the numpy store epilogue on p (then oracle.color_matrix) equals the bytes oracle.scale_and_render writes: one 16 x 16 block
    per colour/alpha pair and all 256 canvas alpha bytes in each, on a 64 x 64-block corner of the GPU frame"""
    src, cv = source(64), canvas(64)
    p = premultiplied(src, linear)
    for name, m in matrices().items():
        exp = cv.copy()
        oracle.scale_and_render(src, exp, filter=24, linear=linear, alpha_meaningful=True, compose=compose, matte=MATTE, color_matrix=m)
        got = wo.composite(p, cv, linear=linear, am=True, compose=compose, matte=MATTE)
        if m is not None:
            oracle.color_matrix(got, m)
        assert np.array_equal(got, exp), (name, int((got != exp).any(-1).sum()))
