"""The chain oracle (tests/color_oracle.py) against hand-derived answers for every ColorFilterSrgb preset and for NaN, infinite, -0.0 and
out-of-range coefficients; EnableTransparency on Bgr32 and Bgra32 frames; and the oracle's RIAPI steps against the product's
riapi_color_steps for every subset of the seven keys.  No GPU is needed."""
import itertools

import numpy as np
import pytest

import imageflow_b200 as ifb
from tests import color_oracle as co

f32 = np.float32


def clamp(v) -> int:
    """color.rs:101-108 uchar_clamp_ff: (v as f64 + 0.5) as i16 as u16, values above 255 -> 0 (v < 0) or 255"""
    v = float(v)
    if v != v:
        return 0
    i = int(max(-32768.0, min(32767.0, np.trunc(v + 0.5))))
    r = i & 0xFFFF
    return (0 if v < 0 else 255) if r > 255 else r


def by_hand(px, m):
    """color_matrix.rs:21-24 on one (b, g, r, a) pixel, written out in f32 with the sums left to right"""
    b, g, r, a = (f32(x) for x in px)
    m = np.asarray(m, f32)
    out = []
    for c in range(4):
        s = m[0, c] * r
        s = f32(s + m[1, c] * g)
        s = f32(s + m[2, c] * b)
        s = f32(s + m[3, c] * a)
        out.append(clamp(f32(s + f32(m[4, c] * f32(255)))))
    r2, g2, b2, a2 = out
    return (b2, g2, r2, a2)


PIXELS = [(0, 0, 0, 0), (255, 255, 255, 255), (10, 20, 30, 40), (200, 100, 50, 128), (1, 254, 127, 0), (77, 3, 250, 255)]


def img_of(pixels):
    return np.array(pixels, np.uint8).reshape(1, -1, 4)


@pytest.mark.parametrize("which", range(10))
@pytest.mark.parametrize("p", [-2.0, -1.0, -0.5, 0.0, 0.1, 0.5, 1.0, 3.0])
def test_each_preset_equals_the_hand_derived_answer(which, p):
    m = co.preset(which, p)[-1][1]
    got, _, _ = co.run_chain(img_of(PIXELS), co.preset(which, p), True)
    assert [tuple(x) for x in got[0]] == [by_hand(px, m) for px in PIXELS]


def test_literal_answers():
    got, _, _ = co.run_chain(img_of([(10, 20, 30, 40)]), co.preset(co.INVERT), True)
    assert tuple(got[0, 0]) == (245, 235, 225, 40)
    got, _, _ = co.run_chain(img_of([(10, 20, 30, 40)]), co.preset(co.BRIGHTNESS, 0.1), True)
    assert tuple(got[0, 0]) == (36, 46, 56, 40)                       # x + 25.5, rounded half up
    got, am, _ = co.run_chain(img_of([(10, 20, 30, 40)]), co.preset(co.ALPHA, 0.5), False)
    assert tuple(got[0, 0]) == (10, 20, 30, 128) and am                # A = 255 first, then 255 * 0.5 = 127.5 -> 128
    got, am, _ = co.run_chain(img_of([(10, 20, 30, 40)]), co.preset(co.ALPHA, 0.5), True)
    assert tuple(got[0, 0]) == (10, 20, 30, 20) and am


@pytest.mark.parametrize("coef,expect", [(np.nan, 0), (np.inf, 255), (-np.inf, 0), (f32(-0.0), 0), (300.0, 255), (-7.5, 0)])
def test_special_coefficients(coef, expect):
    """m[0][0] (red from red) set to the coefficient: NaN clamps to 0, +inf to 255, -inf and negative values to 0; a zero red input
    times inf is NaN (-> 0)"""
    m = np.eye(5, dtype=f32)
    m[0, 0] = coef
    got, _, _ = co.run_chain(img_of([(1, 2, 3, 4), (1, 2, 0, 4)]), [("matrix", m)], True)
    assert got[0, 0, 2] == expect and tuple(got[0, 0, [0, 1, 3]]) == (1, 2, 4)
    assert got[0, 1, 2] == 0                                           # 0 * coefficient: 0, or NaN (-> 0) for +-inf and NaN
    with np.errstate(invalid="ignore"):
        assert [tuple(x) for x in got[0]] == [by_hand(px, m) for px in [(1, 2, 3, 4), (1, 2, 0, 4)]]


def test_enable_transparency_sets_alpha_on_bgr32_only():
    src = img_of([(1, 2, 3, 4), (5, 6, 7, 0)])
    got, am, _ = co.run_chain(src, [("enable_transparency",)], False)
    assert am and (got[..., 3] == 255).all() and (got[..., :3] == src[..., :3]).all()
    got, am, _ = co.run_chain(src, [("enable_transparency",)], True)
    assert am and np.array_equal(got, src)


def test_white_balance_sees_the_frame_as_the_chain_left_it():
    src = np.random.default_rng(1).integers(0, 256, (9, 11, 4), dtype=np.uint8)
    chain = co.preset(co.INVERT) + [("white_balance", None)]
    got, _, hist = co.run_chain(src, chain, True)
    inv, _, _ = co.run_chain(src, co.preset(co.INVERT), True)
    assert np.array_equal(hist, co.histograms(inv))
    want = inv.copy()
    import oracle
    oracle.white_balance(want)
    assert np.array_equal(got, want)


KEYS = {"alpha": 0.4, "brightness": -0.2, "contrast": 0.3, "saturation": -0.5, "sepia": True, "grayscale": "y", "balance_white": "area"}


@pytest.mark.parametrize("subset", [s for r in range(len(KEYS) + 1) for s in itertools.combinations(KEYS, r)], ids=lambda s: "+".join(s) or "none")
def test_riapi_steps_match_the_product_for_every_subset_of_keys(subset):
    kw = {k: KEYS[k] for k in subset}
    want = co.riapi_steps(**kw)
    got = co.of_product(ifb.riapi_color_steps(**kw))
    assert [s[0] for s in got] == [s[0] for s in want]
    for g, w in zip(got, want):
        if g[0] == "matrix":
            assert np.array_equal(g[1].view(np.uint32), np.asarray(w[1], f32).view(np.uint32))
        elif g[0] == "white_balance":
            assert g[1] is None and w[1] is None


@pytest.mark.parametrize("algorithm,which", [("true", co.GRAY_NTSC), ("ntsc", co.GRAY_NTSC), ("y", co.GRAY_NTSC), ("flat", co.GRAY_FLAT),
                                             ("bt709", co.GRAY_BT709), ("ry", co.GRAY_RY)])
def test_grayscale_algorithms(algorithm, which):
    got = co.of_product(ifb.riapi_color_steps(grayscale=algorithm))
    assert len(got) == 1 and np.array_equal(got[0][1], co.preset(which)[0][1])
    assert ifb.riapi_color_steps(balance_white="gimp") == [] and ifb.riapi_color_steps(sepia=False) == []
