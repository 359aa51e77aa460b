"""scale_and_render restated in float64 with a rigorous error bound: for every destination byte, the range [lo, hi] that ANY fp32
evaluation of the same operands could give (TEST INFRASTRUCTURE ONLY; independent of the oracle's resample code).

Restated from the reference: graphics/scaling.rs:55-287 (the store and BlendWithSelf), graphics/color.rs:23-108 (byte->float,
floatspace_to_srgb, uchar_clamp_ff), graphics/lut.rs:4-8 (the 16 K table look-up) and graphics/color_matrix.rs:5-28.  The
operands are taken as given: the contribution windows and weights (oracle.weights), the byte->float tables and the 16 K table,
all of which are pinned to the golden fixtures (tests/test_oracle_golden.py).

  load    p = T[c] * (a * (1/255f)) in float32 (two correctly rounded products: exactly what every implementation computes)
  H       exact sum in f64; any fp32 evaluation of the n_h taps lies within e_H = g(n_h) * sum |w||p|   (g(n) = n u / (1 - n u))
  V       exact sum over exact H in f64; an fp32 evaluation over the fp32 H lies within g(n_v) * sum |v|(|H| + e_H) + sum |v| e_H
  store   interval arithmetic: every fp32 operation widens its result by u * max|endpoint| (+ the subnormal spacing); a branch
          whose condition is undecided on the interval (a > 0, sa > 0.994) takes the union of both outcomes; the encodes are
          monotone, so each byte gets a range [lo, hi]; a colour matrix is evaluated in float32 at the 16 corners of its
          input-byte box (every fp32 operation is monotone in each argument, so the corners hold the extremes).
u = 2^-24.  f64 sums of f32 products carry relative errors near 2^-50, covered by the slack added to u."""
from __future__ import annotations

import numpy as np

import oracle

U = 2.0 ** -24 + 2.0 ** -46          # unit round-off of fp32, plus slack for the f64 evaluation of the exact sums
TINY = 2.0 ** -149                   # absolute error of an operation with a subnormal result
F32 = np.float32
INV255 = F32(1.0) / F32(255.0)       # 1.0f / 255.0f
THR = F32(0.994)


def _gamma(n):
    n = np.asarray(n, np.float64)
    return n * U / (1.0 - n * U)


def _dense(ws, n_in):
    m = np.zeros((len(ws), n_in), np.float64)
    n = np.zeros(len(ws), np.float64)
    for i, (l, r, w) in enumerate(ws):
        m[i, l:r + 1] = w.astype(np.float64)
        n[i] = r - l + 1
    return m, n


class Iv:
    """an interval [lo, hi] of reals (float64 arrays) holding the fp32 value of a quantity"""

    def __init__(self, lo, hi=None):
        self.lo = np.asarray(lo, np.float64)
        self.hi = self.lo if hi is None else np.asarray(hi, np.float64)

    def rounded(self):                                      # one fp32 rounding of anything inside (an exact 0 stays exact)
        m = np.maximum(np.abs(self.lo), np.abs(self.hi))
        e = U * m + np.where(m > 0, TINY, 0.0)
        return Iv(self.lo - e, self.hi + e)

    def __add__(self, o):
        o = _iv(o)
        return Iv(self.lo + o.lo, self.hi + o.hi).rounded()

    def __rsub__(self, c):                                   # c - self
        return Iv(c - self.hi, c - self.lo).rounded()

    def __mul__(self, o):
        o = _iv(o)
        c = np.stack([self.lo * o.lo, self.lo * o.hi, self.hi * o.lo, self.hi * o.hi])
        return Iv(c.min(0), c.max(0)).rounded()

    def div(self, d):
        """self / d.  Where d may be 0 or change sign the quotient is unbounded (a zero numerator still gives 0, or NaN for
        0 / 0, which every encode sends to the byte 0 as well)."""
        one_signed = (d.lo > 0) | (d.hi < 0)
        dl, dh = np.where(one_signed, d.lo, 1.0), np.where(one_signed, d.hi, 1.0)
        c = np.stack([self.lo / dl, self.lo / dh, self.hi / dl, self.hi / dh])
        zero = (self.lo == 0) & (self.hi == 0)
        lo = np.where(one_signed, c.min(0), np.where(zero, 0.0, -np.inf))
        hi = np.where(one_signed, c.max(0), np.where(zero, 0.0, np.inf))
        return Iv(lo, hi).rounded()


def _iv(v):
    return v if isinstance(v, Iv) else Iv(v)


class Bytes:
    """a byte range [lo, hi] (int arrays)"""

    def __init__(self, lo, hi):
        self.lo, self.hi = np.asarray(lo, np.int64), np.asarray(hi, np.int64)

    def union(self, o, take_o):
        """self, widened by o where take_o"""
        return Bytes(np.where(take_o, np.minimum(self.lo, o.lo), self.lo), np.where(take_o, np.maximum(self.hi, o.hi), self.hi))

    def select(self, o, use_o):
        return Bytes(np.where(use_o, o.lo, self.lo), np.where(use_o, o.hi, self.hi))


def _clamp_ff(v):
    """uchar_clamp_ff (color.rs:101-108) of real values: monotone non-decreasing; (v + 0.5) as i16 as u16, > 255 -> 0 or 255"""
    t = np.trunc(np.clip(v, -1e6, 1e6) + 0.5)
    return np.where(t > 255, 255, np.where(t < 0, 0, t)).astype(np.int64)


def _enc(iv: Iv, linear: bool, lut: np.ndarray) -> Bytes:
    """floatspace_to_srgb (color.rs:59-69): linear -> lut16k(v) = LUT[trunc(clamp(v * 16383, 0, 16383))], sRGB space ->
    uchar_clamp_ff(255 v); the product is one fp32 operation"""
    if linear:
        s = iv * 16383.0
        idx = lambda v: np.clip(v, 0.0, 16383.0).astype(np.int64)
        return Bytes(lut[idx(s.lo)], lut[idx(s.hi)])
    s = iv * 255.0
    return Bytes(_clamp_ff(s.lo), _clamp_ff(s.hi))


def _matrix(bgra: list, m: np.ndarray) -> list:
    """color_matrix.rs:5-28 on byte ranges: float32 evaluation at the 16 corners of the (r, g, b, a) box"""
    m = np.asarray(m, np.float32).reshape(5, 5)
    b, g, r, a = bgra
    lo = [np.full(b.lo.shape, 255, np.int64) for _ in range(4)]
    hi = [np.zeros(b.lo.shape, np.int64) for _ in range(4)]
    for corner in range(16):
        fr = (r.hi if corner & 1 else r.lo).astype(np.float32)
        fg = (g.hi if corner & 2 else g.lo).astype(np.float32)
        fb = (b.hi if corner & 4 else b.lo).astype(np.float32)
        fa = (a.hi if corner & 8 else a.lo).astype(np.float32)
        for c in range(4):                                   # output r, g, b, a
            s = m[0, c] * fr + m[1, c] * fg + m[2, c] * fb + m[3, c] * fa + m[4, c] * F32(255.0)
            v = _clamp_ff(s.astype(np.float64))
            lo[c] = np.minimum(lo[c], v); hi[c] = np.maximum(hi[c], v)
    out_r, out_g, out_b, out_a = (Bytes(lo[c], hi[c]) for c in range(4))
    return [out_b, out_g, out_r, out_a]


def byte_ranges(inp: np.ndarray, canvas: np.ndarray, *, x=0, y=0, w=None, h=None, filter=2, sharpen=0.0, linear=True,
                alpha_meaningful=False, compose=0, matte=(0, 0, 0, 0), color_matrix=None):
    """-> (lo, hi): uint8 arrays (h, w, 4) bounding every byte an fp32 evaluation can store into the destination rect of `canvas`
    (which is read, not written)."""
    ih, iw = inp.shape[:2]
    ow = canvas.shape[1] - x if w is None else w
    oh = canvas.shape[0] - y if h is None else h
    am = bool(alpha_meaningful)
    lobe = oracle.LOBE_SHARPEN_PERCENT if sharpen > 0.0 else oracle.LOBE_NATURAL
    Wv, nv = _dense(oracle.weights(filter, oh, ih, 1.0, lobe, sharpen), ih)
    Wh, nh = _dense(oracle.weights(filter, ow, iw, 1.0, lobe, sharpen), iw)
    T = oracle.byte_to_float_table(linear)
    lut = oracle.linear_to_srgb_table().astype(np.int64)

    # ---- load (exact: the same two roundings everywhere)
    px = np.ascontiguousarray(inp)
    nch = 4 if am else 3
    if am:
        af = px[..., 3].astype(np.float32) * INV255
        p = np.empty((ih, iw, 4), np.float32)
        for c in range(3):
            p[..., c] = T[px[..., c]] * af
        p[..., 3] = af
    else:
        p = T[px[..., :3]]
    p = p.astype(np.float64)

    # ---- H and V sums with their bounds: (ih, iw, c) -> (ih, ow, c) -> (oh, ow, c)
    H = np.einsum("jkc,Xk->jXc", p, Wh, optimize=True)
    eH = _gamma(nh)[None, :, None] * np.einsum("jkc,Xk->jXc", np.abs(p), np.abs(Wh), optimize=True)
    F = np.einsum("jXc,yj->yXc", H, Wv, optimize=True)
    aWv = np.abs(Wv)
    eV = _gamma(nv)[:, None, None] * np.einsum("jXc,yj->yXc", np.abs(H) + eH, aWv, optimize=True) \
        + np.einsum("jXc,yj->yXc", eH, aWv, optimize=True)
    ch = [Iv(F[..., c] - eV[..., c], F[..., c] + eV[..., c]) for c in range(nch)]

    # ---- store (scaling.rs)
    cv = np.ascontiguousarray(canvas)[y:y + oh, x:x + ow]
    if not am:                                               # scaling.rs:227-232, and the !alpha_meaningful arm of BlendWithSelf
        out = [_enc(ch[c], linear, lut) for c in range(3)] + [Bytes(np.full((oh, ow), 255), np.full((oh, ow), 255))]
    elif compose == oracle.BLEND_WITH_SELF:                  # scaling.rs:254-287
        sa = ch[3]
        opaque_may, blend_may = sa.hi > THR, sa.lo <= THR
        da = cv[..., 3].astype(np.float32)
        k = Iv((INV255 * da).astype(np.float64))             # dest_alpha_coeff * da + 0.0: one exact-valued constant per pixel
        dc = (1.0 - sa) * k
        fa = sa + dc                                         # 0 over an alpha-0 canvas pixel when sa == 0; negative when sa < 0
        fa255 = fa * 255.0
        a_bytes = Bytes(_clamp_ff(fa255.lo), _clamp_ff(fa255.hi))
        out = []
        for c in range(3):
            num = ch[c] + dc * T[cv[..., c]].astype(np.float64)
            e = _enc(num.div(fa), linear, lut)
            direct = _enc(ch[c], linear, lut)
            out.append(direct.select(e, blend_may & ~opaque_may).union(e, blend_may & opaque_may))
        opaque_a = Bytes(np.full((oh, ow), 255), np.full((oh, ow), 255))
        out.append(opaque_a.select(a_bytes, blend_may & ~opaque_may).union(a_bytes, blend_may & opaque_may))
    else:                                                    # ReplaceSelf / BlendWithMatte with meaningful alpha
        b, g, r, a = ch
        if compose == oracle.BLEND_WITH_MATTE:               # scaling.rs:119-148: the matte premultiplied in working space
            ma = F32(matte[3]) * INV255
            mt = [T[matte[c]] * ma for c in range(3)] + [ma]
            t = 1.0 - a
            b, g, r, a = (v + t * float(mt[c]) for c, v in enumerate((b, g, r, a)))
        div_may, keep_may = a.hi > 0, a.lo <= 0
        out = []
        for v in (b, g, r):
            q = _enc(v.div(a), linear, lut)
            direct = _enc(v, linear, lut)
            out.append(direct.select(q, div_may & ~keep_may).union(q, div_may & keep_may))
        a255 = a * 255.0
        out.append(Bytes(_clamp_ff(a255.lo), _clamp_ff(a255.hi)))
    if color_matrix is not None:
        out = _matrix(out, color_matrix)
    lo = np.stack([np.broadcast_to(o.lo, (oh, ow)) for o in out], -1).astype(np.uint8)
    hi = np.stack([np.broadcast_to(o.hi, (oh, ow)) for o in out], -1).astype(np.uint8)
    return lo, hi
