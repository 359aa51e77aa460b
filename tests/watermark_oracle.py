"""CPU oracles of the Watermark node (TEST INFRASTRUCTURE): the node-by-node expansion of flow/nodes/watermark.rs (copy of the
cropped watermark, ColorFilterSrgb::Alpha through the colour oracle, DrawImageExact through oracle.scale_and_render under the Compose
rule), and the composite of a resampled F (oracle.resample_stages) over a canvas rectangle -- the store epilogue of the resample
(finish_pixel, ifb_finish.cuh; scaling.rs:227-287) restated in numpy float32."""
import numpy as np

import oracle
from tests import color_oracle as co

REPLACE_SELF, BLEND_WITH_SELF, BLEND_WITH_MATTE = 0, 1, 2
_F = np.float32


def drawn_compose(compose: int) -> int:
    """scale_render.rs:282-284: a ReplaceSelf canvas is drawn on as BlendWithSelf under CompositingMode::Compose"""
    return BLEND_WITH_SELF if compose == REPLACE_SELF else compose


def source_of(wm: np.ndarray, wm_am: bool, draw):
    """the watermark bitmap the DrawImageExact of `draw` reads: the crop (a copy), then the Alpha filter -> (pixels, alpha_meaningful)"""
    src = wm if draw.crop is None else wm[draw.crop[1]:draw.crop[3], draw.crop[0]:draw.crop[2]]
    src = np.ascontiguousarray(src).copy()
    if draw.opacity is None:
        return src, bool(wm_am)
    out, am, _ = co.run_chain(src, co.preset(co.ALPHA, draw.opacity), wm_am)
    return out, am


def expansion(frame: np.ndarray, frame_compose: int, matte, wm: np.ndarray, wm_am: bool, draw) -> None:
    """the node-by-node expansion of one Watermark on `frame` (h, w, 4), in place"""
    src, am = source_of(wm, wm_am, draw)
    oracle.scale_and_render(src, frame, x=draw.x, y=draw.y, w=draw.w, h=draw.h, filter=int(draw.filter), linear=True,
                            alpha_meaningful=am, compose=drawn_compose(frame_compose), matte=tuple(matte))


def f_of(src: np.ndarray, am: bool, w: int, h: int, filter: int, linear: bool = True, sharpen: float = 0.0) -> np.ndarray:
    """F: the resampled premultiplied working-space image (h, w, 4) float32, as oracle.resample_stages leaves it"""
    scratch = np.zeros((h, w, 4), np.uint8)
    _, f = oracle.resample_stages(src, scratch, filter=filter, linear=linear, alpha_meaningful=am, sharpen=sharpen)
    return f


def _clamp_ff(x):
    """color.rs:101-108 uchar_clamp_ff on float32 arrays (NaN -> 0)"""
    with np.errstate(invalid="ignore"):
        fl = np.floor(x)
        v = fl + ((x - fl) >= _F(0.5))
        v = np.where(x >= _F(255), _F(255), v)
        v = np.where(x > _F(0), v, _F(0))
    return v.astype(np.uint8)


def composite(f: np.ndarray, dst: np.ndarray, *, linear: bool, am: bool, compose: int, matte=(0, 0, 0, 0)) -> np.ndarray:
    """finish_pixel(F, dst) for every pixel: the bytes the store writes (dst is read for BlendWithSelf only)"""
    T = oracle.byte_to_float_table(linear)
    lut = oracle.linear_to_srgb_table()

    def enc(v):
        if not linear:
            return _clamp_ff(_F(255) * v)
        with np.errstate(invalid="ignore"):
            s = np.nan_to_num(np.clip(v * _F(16383), _F(0), _F(16383)), nan=0.0)
        return lut[s.astype(np.int64)]

    b, g, r, a = (f[..., i].astype(_F) for i in range(4))
    out = np.empty(f.shape[:2] + (4,), np.uint8)
    with np.errstate(all="ignore"):
        if compose == BLEND_WITH_SELF:
            da = dst[..., 3].astype(_F)
            dc = (_F(1) - a) * ((_F(1.0 / 255.0) * da) + _F(0))
            fa = a + dc
            blend = [enc((c + dc * T[dst[..., k]]) / fa) for k, c in enumerate((b, g, r))]
            plain = [enc(c) for c in (b, g, r)]
            keep = (a > _F(0.994)) | (not am)
            for k in range(3):
                out[..., k] = np.where(keep, plain[k], blend[k])
            out[..., 3] = np.where(keep, 255, _clamp_ff(fa * _F(255)))
        elif not am:
            for k, c in enumerate((b, g, r)):
                out[..., k] = enc(c)
            out[..., 3] = 255
        else:
            if compose == BLEND_WITH_MATTE:
                tb = oracle.byte_to_float_table(linear)
                ma = _F(matte[3]) * _F(1.0 / 255.0)
                mt = [_F(tb[matte[k]]) * ma for k in range(3)] + [ma]
                t = _F(1) - a
                b, g, r, a = b + t * mt[0], g + t * mt[1], r + t * mt[2], a + t * mt[3]
            pos = a > _F(0)
            b, g, r = (np.where(pos, c / np.where(pos, a, _F(1)), c) for c in (b, g, r))
            for k, c in enumerate((b, g, r)):
                out[..., k] = enc(c)
            out[..., 3] = _clamp_ff(a * _F(255))
    return out
