"""Pixel-format conversions restated in numpy from the reference (test oracle): the row swizzles of graphics/swizzle.rs:8-45 and the RGB
rows of Bitmap::to_vec_rgb (graphics/bitmaps.rs:1316-1345), on (H, W, C) uint8 arrays.  Ops are numbered as enum ifb200_pixel_op
(include/ifb200.h); `opaque` writes 255 into every alpha byte of a 4-byte output."""
import numpy as np

RGB24_TO_BGRA, RGBA_TO_BGRA, GRAY_TO_BGRA, GRAY_ALPHA_TO_BGRA, BGRA_TO_RGB24 = range(5)
OPS = (RGB24_TO_BGRA, RGBA_TO_BGRA, GRAY_TO_BGRA, GRAY_ALPHA_TO_BGRA, BGRA_TO_RGB24)
CHANNELS = {RGB24_TO_BGRA: (3, 4), RGBA_TO_BGRA: (4, 4), GRAY_TO_BGRA: (1, 4), GRAY_ALPHA_TO_BGRA: (2, 4), BGRA_TO_RGB24: (4, 3)}


def rgb_to_bgra(src):
    """rgb_to_bgra: 3 source bytes -> 4, alpha 255"""
    h, w, _ = src.shape
    out = np.empty((h, w, 4), np.uint8)
    out[..., 0], out[..., 1], out[..., 2], out[..., 3] = src[..., 2], src[..., 1], src[..., 0], 255
    return out


def copy_swap_br(src):
    """copy_swap_br: bytes 0 and 2 swapped, alpha copied (BGRA <-> RGBA)"""
    return np.ascontiguousarray(src[..., [2, 1, 0, 3]])


def gray_to_bgra(src):
    """gray_to_bgra: R = G = B = gray, A = 255"""
    v = src[..., 0]
    return np.stack([v, v, v, np.full_like(v, 255)], axis=-1)


def gray_alpha_to_bgra(src):
    """gray_alpha_to_bgra: R = G = B = gray, A = alpha"""
    v = src[..., 0]
    return np.stack([v, v, v, src[..., 1]], axis=-1)


def to_vec_rgb(src):
    """to_vec_rgb: RGB8 { r: pix.r, g: pix.g, b: pix.b } of each BGRA pixel; alpha dropped, no matte"""
    return np.ascontiguousarray(src[..., [2, 1, 0]])


_FN = {RGB24_TO_BGRA: rgb_to_bgra, RGBA_TO_BGRA: copy_swap_br, GRAY_TO_BGRA: gray_to_bgra, GRAY_ALPHA_TO_BGRA: gray_alpha_to_bgra,
       BGRA_TO_RGB24: to_vec_rgb}


def convert(op, src, opaque=False):
    """the destination rows of `op` on the (H, W, C) source rows"""
    out = _FN[op](np.asarray(src, np.uint8))
    if opaque and out.shape[2] == 4:
        out = out.copy()
        out[..., 3] = 255
    return out
