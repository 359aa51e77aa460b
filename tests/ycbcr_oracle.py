"""CPU reference of ifb200_batch_ycbcr_to_bgra: libjpeg-turbo's decoder colour stage restated in numpy integers (jdsample.c's
upsamplers as JCS_EXT_BGRA output selects them under the default do_fancy_upsampling, then jdcolor.c's ycc_rgb_convert tables).  Test
infrastructure: tests/golden/ycbcr_golden.npz holds libjpeg-turbo's own output, which tests/test_ycbcr_oracle.py compares against this.

Per pixel, with y, cb, cr the planes' samples after upsampling to w x h:
  R = clamp(y + ((FIX(1.40200) (cr - 128) + ONE_HALF) >> 16))
  G = clamp(y + ((-FIX(0.34414) (cb - 128) + ONE_HALF - FIX(0.71414) (cr - 128)) >> 16))
  B = clamp(y + ((FIX(1.77200) (cb - 128) + ONE_HALF) >> 16))
  FIX(x) = int(x * 65536 + 0.5), ONE_HALF = 1 << 15, >> arithmetic, clamp to 0..255; output (B, G, R, 255).
Upsampling of a chroma plane (cw x ch) to w x h, neighbour indices clamped to the plane (the first and last rows and columns repeated):
  4:4:4  none.
  4:2:2  cw = ceil(w / 2).  Output column 2i = (3 c[i] + c[i - 1] + 1) >> 2, column 2i + 1 = (3 c[i] + c[i + 1] + 2) >> 2 (h2v1).
  4:2:0  cw = ceil(w / 2), ch = ceil(h / 2).  Column sums s[j][i] = 3 c[j][i] + c[j -/+ 1][i] for output row 2j / 2j + 1, then
         output column 2i = (3 s[i] + s[i - 1] + 8) >> 4, column 2i + 1 = (3 s[i] + s[i + 1] + 7) >> 4 (h2v2).
  libjpeg-turbo runs the fancy forms only when cw > 2; a plane one or two columns wide is replicated (h2v1_upsample / h2v2_upsample):
  every output pixel takes c[y >> 1 (4:2:0) or y][x >> 1].  Both cases are the formulas above with the weights (4, 0) for (3, 1).
Then cropped to w x h."""
import numpy as np

S444, S422, S420 = 0, 1, 2
SAMPLINGS = (S444, S422, S420)
NAMES = {S444: "444", S422: "422", S420: "420"}

FIX_CR_R, FIX_CB_B, FIX_CR_G, FIX_CB_G = 91881, 116130, 46802, 22554   # FIX(1.40200), FIX(1.77200), FIX(0.71414), FIX(0.34414)
ONE_HALF = 1 << 15


def chroma_shape(sampling, w, h):
    """(rows, columns) of a chroma plane of a w x h frame"""
    if sampling == S444:
        return h, w
    return ((h + 1) // 2 if sampling == S420 else h), (w + 1) // 2


def _h2(c, w, bias_even, bias_odd, shift):
    """horizontal 2x of columns c (int64, last axis) to w columns: (a c[i] + b c[i -/+ 1] + bias) >> shift"""
    n = c.shape[-1]
    a, b = (3, 1) if n > 2 else (4, 0)
    left = np.concatenate([c[..., :1], c[..., :-1]], axis=-1)
    right = np.concatenate([c[..., 1:], c[..., -1:]], axis=-1)
    out = np.empty(c.shape[:-1] + (2 * n,), np.int64)
    out[..., 0::2] = (a * c + b * left + bias_even) >> shift
    out[..., 1::2] = (a * c + b * right + bias_odd) >> shift
    return out[..., :w]


def upsample(sampling, plane, w, h):
    """the chroma plane (ch x cw, uint8) at w x h, as libjpeg-turbo's upsampler gives it (int64)"""
    c = np.asarray(plane, np.int64)
    assert c.shape == chroma_shape(sampling, w, h), (c.shape, chroma_shape(sampling, w, h))
    if sampling == S444:
        return c
    if sampling == S422:
        return _h2(c, w, 1, 2, 2)
    a, b = (3, 1) if c.shape[1] > 2 else (4, 0)
    above = np.concatenate([c[:1], c[:-1]], axis=0)
    below = np.concatenate([c[1:], c[-1:]], axis=0)
    s = np.empty((2 * c.shape[0], c.shape[1]), np.int64)
    s[0::2] = a * c + b * above
    s[1::2] = a * c + b * below
    return _h2(s[:h], w, 8, 7, 4)


def ycc_to_bgra(y, cb, cr):
    """full-resolution samples (any integer arrays of one shape) -> (..., 4) uint8 BGRA, alpha 255"""
    y, cb, cr = (np.asarray(v, np.int64) for v in (y, cb, cr))
    cb, cr = cb - 128, cr - 128
    r = y + ((FIX_CR_R * cr + ONE_HALF) >> 16)
    g = y + ((-FIX_CB_G * cb + ONE_HALF - FIX_CR_G * cr) >> 16)
    b = y + ((FIX_CB_B * cb + ONE_HALF) >> 16)
    out = np.empty(y.shape + (4,), np.uint8)
    out[..., 0], out[..., 1], out[..., 2] = (np.clip(v, 0, 255) for v in (b, g, r))
    out[..., 3] = 255
    return out


def convert(sampling, y, cb, cr):
    """(h, w) luma and the two chroma planes at their subsampled size -> (h, w, 4) BGRA as JCS_EXT_BGRA decodes them"""
    y = np.asarray(y)
    h, w = y.shape
    return ycc_to_bgra(y, upsample(sampling, cb, w, h), upsample(sampling, cr, w, h))
