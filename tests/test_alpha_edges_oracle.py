"""The store epilogue's alpha edges, on the CPU: content that reaches them, and a float64 reference that bounds the oracle there.

Transparent inputs (logos, cut-outs) give filtered alphas that noise never does: exactly 0 over the transparent field, slightly
negative or above 1 next to hard edges (negative lobes), tiny positive tails, values next to BlendWithSelf's 0.994 threshold,
and -- composited over an alpha-0 canvas pixel -- fa == 0 (0 / 0, NaN, byte 0) or fa < 0.  Every kernel's store epilogue
branches on exactly these values (scaling.rs:55-88, 254-287).
  * test_cutout_content_reaches_every_alpha_class: each cut-out case reaches the classes its comment names (a later edit to the
    content that stops reaching one fails here, not silently in the GPU tests).
  * test_oracle_inside_f64_ranges: every byte of the oracle lies in the range that tests/resample_f64.py (an independent
    float64 restatement with a rigorous fp32 error bound) allows, and the bytes that range pins down are equal; the fraction of
    bytes left undecided is printed and held under a measured limit so that the check cannot quietly become vacuous."""
import numpy as np
import pytest

import oracle
from imageflow_b200 import synth
from tests import resample_f64, util

# (in_w, in_h, out_w, out_h, filter, alpha classes the V-pass alpha reaches)
ALL = ("a==0", "a<0", "0<a<1e-4", "a>1", "|a-0.994|<1e-3", "fa==0", "fa<0")
CUTOUT = [
    (640, 480, 200, 150, 2, ALL),                                            # Robidoux 3.2x (config-1 ratio)
    (512, 384, 128, 96, 2, ALL),                                             # Robidoux 4x
    (960, 540, 128, 128, 6, ("a<0", "0<a<1e-4", "a>1", "|a-0.994|<1e-3", "fa<0")),   # Lanczos3 at config-2 ratios: ring depth 6
    (100, 60, 333, 200, 14, ALL),                                            # Mitchell 3.3x up-scale (tile kernel)
    (300, 200, 300, 200, 2, ("a==0", "|a-0.994|<1e-3", "fa==0")),            # 1:1 (Robidoux has no negative taps at 1:1)
]
MATTE = (40, 120, 250, 200)          # alpha below 255: BlendWithMatte leaves partial alpha


def _classes(a, fa, blend):
    return {"a==0": a == 0, "a<0": a < 0, "0<a<1e-4": (a > 0) & (a < 1e-4), "a>1": a > 1,
            "|a-0.994|<1e-3": np.abs(a.astype(np.float64) - 0.994) < 1e-3, "fa==0": blend & (fa == 0), "fa<0": blend & (fa < 0)}


def _id(c):
    return "x".join(map(str, c[:5]))


def test_cutout_numpy_and_torch_give_the_same_bytes():
    for (w, h, seed) in ((333, 201, 5), (64, 64, 0), (7, 3, 9)):
        assert np.array_equal(synth.cutout_np(w, h, seed), synth.cutout_torch(w, h, seed, device="cpu").numpy())
        assert np.array_equal(synth.cutout_canvas_np(w, h, seed), synth.cutout_canvas_torch(w, h, seed, device="cpu").numpy())
    a = synth.cutout_np(640, 480, 1)
    assert (a[..., :3][a[..., 3] == 0] != 0).all()                     # colour under alpha 0 is never 0
    counts = np.bincount(a[..., 3].ravel(), minlength=256)
    assert counts[0] > 0.4 * a[..., 3].size and counts[253] > 0 and counts[254] > 0 and counts[255] > 0
    assert set(np.unique(a[..., 3])) == {0, 253, 254, 255}
    cv = synth.cutout_canvas_np(200, 150, 3)
    assert (cv[..., 3] == 0).mean() > 0.25 and (cv[..., 3] == 255).mean() > 0.25


@pytest.mark.parametrize("case", CUTOUT, ids=_id)
def test_cutout_content_reaches_every_alpha_class(case):
    iw, ih, ow, oh, flt, want = case
    inp = synth.cutout_np(iw, ih, seed=iw + oh)
    cv = synth.cutout_canvas_np(ow, oh, seed=3)
    _, F = oracle.resample_stages(inp, cv.copy(), filter=flt, alpha_meaningful=True)
    a = F[..., 3]                                                       # the V-pass alpha, before the store
    k = np.float32(1.0) / np.float32(255.0)
    fa = a + (np.float32(1.0) - a) * (k * cv[..., 3].astype(np.float32))   # BlendWithSelf's final alpha
    got = {name: int(m.sum()) for name, m in _classes(a, fa, a <= np.float32(0.994)).items()}
    print(_id(case), got)
    missing = [c for c in want if got[c] == 0]
    assert not missing, (case[:5], missing, got)


def _variants():
    sepia, general = oracle.color_filter_matrix(0), oracle.color_filter_matrix(6, 0.5)
    general = general.copy()
    general[4, 0] = 0.1
    # (alpha meaningful, linear, compose, colour matrix, sharpen)
    return [(True, True, 0, None, 0.0), (True, True, 1, None, 0.0), (True, True, 2, None, 0.0), (True, False, 1, sepia, 0.0),
            (True, False, 2, None, 0.0), (True, True, 1, general, 0.0), (False, True, 0, None, 0.0), (True, True, 0, None, 30.0)]


NOISE = [                             # tests/test_order_band.py's geometries
    (640, 480, 200, 150, 2), (960, 540, 128, 128, 6), (512, 384, 128, 96, 14), (200, 150, 400, 300, 14), (300, 200, 300, 200, 2),
]
F64_CASES = [("cutout",) + c[:5] + (vi,) for c in CUTOUT for vi in range(len(_variants()))] + \
            [("noise",) + c + (vi,) for c in NOISE for vi in range(len(_variants()))]
# Largest fraction of bytes whose f64 range is wider than one value.  Measured worst cases: 4.1e-2 (cut-out, sRGB space: the
# quotient by a tiny alpha), 4.0e-3 (noise, Lanczos3 7.5x); the limits are twice that, so ranges gone vacuous would fail.
AMBIGUOUS_LIMIT = {"cutout": 0.08, "noise": 0.008}


def f64_frame(kind, iw, ih, ow, oh, seed):
    if kind == "cutout":
        return synth.cutout_np(iw, ih, seed=seed), synth.cutout_canvas_np(ow + 5, oh + 3, seed=seed + 1)
    return util.noise(iw, ih, seed=seed, alpha_mode="mixed"), util.noise(ow + 5, oh + 3, seed=seed + 1, alpha_mode="mixed")


def check_inside_ranges(got, lo, hi):
    """-> fraction of undecided bytes; asserts 100 % inside [lo, hi]"""
    out = (got < lo) | (got > hi)
    assert not out.any(), (int(out.sum()), np.argwhere(out)[:5].tolist(), got[out][:8].tolist(), lo[out][:8].tolist(), hi[out][:8].tolist())
    return float((lo != hi).mean())


def test_linear_to_srgb_table_is_monotone():
    """the ranges rely on the encodes being monotone"""
    assert (np.diff(oracle.linear_to_srgb_table().astype(np.int16)) >= 0).all()


@pytest.mark.parametrize("case", F64_CASES, ids=lambda c: f"{c[0]}-{'x'.join(map(str, c[1:6]))}-v{c[6]}")
def test_oracle_inside_f64_ranges(case):
    kind, iw, ih, ow, oh, flt, vi = case
    alpha, linear, compose, cm, sharpen = _variants()[vi]
    inp, canvas = f64_frame(kind, iw, ih, ow, oh, seed=iw + oh + vi)
    if not alpha:
        inp = inp.copy(); inp[..., 3] = 255
    kw = dict(x=2, y=1, w=ow, h=oh, filter=flt, sharpen=sharpen, linear=linear, alpha_meaningful=alpha, compose=compose,
              matte=MATTE, color_matrix=cm)
    exp = canvas.copy()
    oracle.scale_and_render(inp, exp, **kw)
    lo, hi = resample_f64.byte_ranges(inp, canvas, **kw)
    frac = check_inside_ranges(exp[1:1 + oh, 2:2 + ow], lo, hi)
    print(f"{kind} {iw}x{ih}->{ow}x{oh} f{flt} alpha={alpha} linear={linear} compose={compose} cm={cm is not None} "
          f"sharpen={sharpen}: ambiguous {frac:.2e}")
    assert frac <= AMBIGUOUS_LIMIT[kind], frac
