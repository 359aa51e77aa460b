"""CPU reference of ifb200_batch_bgra_to_ycbcr: libjpeg-turbo's compressor colour stage restated in numpy integers (jccolor.c's
rgb_ycc_convert, then jcsample.c's downsamplers with the edge expansion in front of them), after apply_matte when alpha is meaningful.
Test infrastructure: tests/golden/ycbcr_enc_golden.npz holds cases pinned against libjpeg-turbo itself, which
tests/test_ycbcr_enc_oracle.py compares against this.

Per pixel, FIX(x) = int(x * 65536 + 0.5), >> arithmetic (every result lies in 0..255, no clamp):
  Y  = (FIX(0.29900) R + FIX(0.58700) G + FIX(0.11400) B + ONE_HALF) >> 16
  Cb = (-FIX(0.16874) R - FIX(0.33126) G + FIX(0.5) B + (128 << 16) + ONE_HALF - 1) >> 16
  Cr = (FIX(0.5) R - FIX(0.41869) G - FIX(0.08131) B + (128 << 16) + ONE_HALF - 1) >> 16
Downsampling of the full-resolution Cb and Cr, after the last column and row are replicated to an even width and height:
  4:4:4  a copy.
  4:2:2  column i = (c[2i] + c[2i + 1] + bias) >> 1, bias 0, 1, 0, 1, ... from column 0 (h2v1_downsample).
  4:2:0  sample (i, j) = (c[2j][2i] + c[2j][2i + 1] + c[2j + 1][2i] + c[2j + 1][2i + 1] + bias) >> 2, bias 1, 2, 1, 2, ... from
         column 0 (h2v2_downsample).
Only the visible samples are kept: ceil(w / 2) columns, and ceil(h / 2) rows at 4:2:0."""
import numpy as np

from tests.ycbcr_oracle import NAMES, S420, S422, S444, SAMPLINGS, chroma_shape  # noqa: F401  (re-exported)

ONE_HALF = 1 << 15


def rgb_to_ycc(bgra):
    """(Y, Cb, Cr) int64 planes of a (H, W, 4 or 3) BGRA array; alpha is ignored, as libjpeg ignores it in JCS_EXT_BGRA"""
    b, g, r = (bgra[..., c].astype(np.int64) for c in (0, 1, 2))
    y = (19595 * r + 38470 * g + 7471 * b + ONE_HALF) >> 16
    cb = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + ONE_HALF - 1) >> 16
    cr = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + ONE_HALF - 1) >> 16
    return y, cb, cr


def downsample(sampling, c):
    """a full-resolution chroma plane (int64, H x W) at `sampling`, as uint8"""
    if sampling == S444:
        return c.astype(np.uint8)
    h, w = c.shape
    c = np.pad(c, ((0, h % 2 if sampling == S420 else 0), (0, w % 2)), mode="edge")
    cols = c.shape[1] // 2
    if sampling == S422:
        bias = np.arange(cols) & 1
        return ((c[:, 0::2] + c[:, 1::2] + bias) >> 1).astype(np.uint8)
    bias = 1 + (np.arange(cols) & 1)
    return ((c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2] + bias) >> 2).astype(np.uint8)


def convert(sampling, bgra):
    """(y, cb, cr) uint8 planes of an opaque (or already flattened) (H, W, 4) BGRA frame"""
    y, cb, cr = rgb_to_ycc(bgra)
    return y.astype(np.uint8), downsample(sampling, cb), downsample(sampling, cr)


def flatten(bgra, matte_bgra, alpha_meaningful):
    """apply_matte (graphics/blend.rs) on a copy, through the CPU oracle of ifb200_apply_matte_bgra8"""
    import oracle
    out = np.ascontiguousarray(bgra).copy()
    oracle.apply_matte(out, matte_bgra, alpha_meaningful)
    return out


def convert_matte(sampling, bgra, matte_bgra=(255, 255, 255, 255), alpha_meaningful=True):
    """ifb200_batch_bgra_to_ycbcr of one frame: the planes of flatten(bgra) (or of bgra itself when alpha is not meaningful)"""
    return convert(sampling, flatten(bgra, matte_bgra, alpha_meaningful) if alpha_meaningful else bgra)
