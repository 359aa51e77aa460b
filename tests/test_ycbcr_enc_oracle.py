"""tests/ycbcr_enc_oracle.py, the numpy restatement of libjpeg-turbo's compressor colour stage, against libjpeg-turbo itself: every case
of tests/golden/ycbcr_enc_golden.npz (written by tests/golden/make_ycbcr_enc_golden.py with Pillow's bundled libjpeg-turbo, which pins
each case through JPEG streams) byte for byte, the matte cases through the CPU oracle of apply_matte.  No GPU is needed."""
import os

import numpy as np
import pytest

from tests import ycbcr_enc_oracle as eo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ycbcr_enc_golden.npz")
_Z = np.load(GOLDEN)
CASES = [str(c) for c in _Z["cases"]]
MATTE = tuple(int(v) for v in _Z["matte_bgra"])
SAMPLING_OF = {v: k for k, v in eo.NAMES.items()}


def golden_case(name):
    """(sampling, BGRA source, y, cb, cr, matte case?) of one fixture case; a matte case is flattened over MATTE"""
    return ((SAMPLING_OF[name.split("_")[0]],) + tuple(_Z[f"{name}/{k}"] for k in ("bgra", "y", "cb", "cr")) + (name.endswith("m"),))


@pytest.mark.parametrize("name", CASES)
def test_oracle_equals_libjpeg_turbo(name):
    s, src, y, cb, cr, matte = golden_case(name)
    h, w = src.shape[:2]
    assert y.shape == (h, w) and cb.shape == cr.shape == eo.chroma_shape(s, w, h)
    got = eo.convert_matte(s, src, MATTE, True) if matte else eo.convert(s, src)
    for g, want, plane in zip(got, (y, cb, cr), ("Y", "Cb", "Cr")):
        assert np.array_equal(g, want), (plane, np.argwhere(g != want)[:4].tolist())


def test_the_fixture_covers_what_it_pins():
    """all three samplings at aligned and ragged sizes, 1x1, 1xN and Nx1, odd widths and heights, cut-out alpha over a matte, and
    libjpeg-turbo's version"""
    assert str(_Z["libjpeg_turbo_version"]).startswith("3.")
    sizes, mattes = {}, {}
    for name in CASES:
        s, src, *_, matte = golden_case(name)
        (mattes if matte else sizes).setdefault(s, set()).add(src.shape[1::-1])
    for s in eo.SAMPLINGS:
        assert len(sizes[s]) >= 15 and len(mattes[s]) >= 2, (s, sizes[s], mattes[s])
        assert {(16, 16), (240, 32), (250, 33)} <= sizes[s]
        assert any(w % 2 and h % 2 for w, h in sizes[s]) and any(w == 1 and h > 1 for w, h in sizes[s]) and any(h == 1 for _, h in sizes[s])
    alpha = np.concatenate([golden_case(n)[1][..., 3].ravel() for n in CASES if n.endswith("m")])
    assert (alpha == 0).any() and (alpha == 255).any() and ((alpha > 0) & (alpha < 255)).any()
    # the cases the stream checks could not pin are named, with the reasons in the generator's docstring
    assert not set(CASES) & set(str(d) for d in _Z["dropped"])


def test_hand_derived_values():
    """jccolor.c at a few points: gray is neutral chroma, the primaries reach the ends without a clamp"""
    px = np.array([[[0, 0, 0, 255], [128, 128, 128, 255], [255, 255, 255, 255], [255, 0, 0, 255], [0, 0, 255, 255]]], np.uint8)
    y, cb, cr = (p[0].tolist() for p in eo.convert(eo.S444, px))
    assert y == [0, 128, 255, 29, 76] and cb[:3] == [128] * 3 and cr[:3] == [128] * 3
    # blue: Cb = (32768 * 255 + 8388608 + 32767) >> 16 = 255; red: Cr = 255 and Cb = (-11059 * 255 + 8421375) >> 16 = 85
    assert cb[3] == 255 and cr[4] == 255 and cb[4] == 85


def test_downsampling_by_hand():
    """h2v1 and h2v2 biases alternate with the output column from 0 (1 at 4:2:0); the last odd column and row are replicated"""
    c = np.array([[0, 1, 1, 2, 5]])
    assert eo.downsample(eo.S422, c).tolist() == [[0, 2, 5]]        # (0+1+0)>>1, (1+2+1)>>1, (5+5+0)>>1
    c2 = np.array([[0, 1, 2, 2, 7], [1, 1, 1, 2, 8]])
    assert eo.downsample(eo.S420, c2).tolist() == [[(0 + 1 + 1 + 1 + 1) >> 2, (2 + 2 + 1 + 2 + 2) >> 2, (2 * (7 + 8) + 1) >> 2]]
    assert eo.downsample(eo.S420, np.array([[3, 4, 9]])).tolist() == [[(2 * 7 + 1) >> 2, (4 * 9 + 2) >> 2]]
