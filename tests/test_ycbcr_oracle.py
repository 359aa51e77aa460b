"""tests/ycbcr_oracle.py, the numpy restatement of libjpeg-turbo's decoder colour stage, against libjpeg-turbo itself: every case of
tests/golden/ycbcr_golden.npz (written by tests/golden/make_ycbcr_golden.py with Pillow's bundled libjpeg-turbo) byte for byte.  The
fixture's 4:2:2 planes are solved preimages of libjpeg-turbo's h2v1 upsampling, so 4:2:2 is pinned more weakly than 4:4:4 and 4:2:0,
whose planes are decoder output.  No GPU is needed."""
import os

import numpy as np
import pytest

from tests import ycbcr_oracle as yo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ycbcr_golden.npz")
_Z = np.load(GOLDEN)
CASES = [str(c) for c in _Z["cases"]]
SAMPLING_OF = {v: k for k, v in yo.NAMES.items()}


def golden_case(name):
    """(sampling, y, cb, cr, expected BGRA) of one fixture case"""
    return (SAMPLING_OF[name.split("_")[0]],) + tuple(_Z[f"{name}/{k}"] for k in ("y", "cb", "cr", "bgra"))


@pytest.mark.parametrize("name", CASES)
def test_oracle_equals_libjpeg_turbo(name):
    s, y, cb, cr, want = golden_case(name)
    assert cb.shape == cr.shape == yo.chroma_shape(s, y.shape[1], y.shape[0])
    got = yo.convert(s, y, cb, cr)
    assert np.array_equal(got, want), np.argwhere(np.any(got != want, axis=2))[:4].tolist()


def test_the_fixture_covers_what_it_pins():
    """all three samplings at about 20 sizes, 1x1, 1xN and Nx1, chroma planes one and two columns wide, and libjpeg-turbo's version"""
    assert str(_Z["libjpeg_turbo_version"]).startswith("3.")
    sizes = {}
    for name in CASES:
        s, y, *_ = golden_case(name)
        sizes.setdefault(s, set()).add(y.shape[::-1])
    assert all(len(sizes[s]) >= 20 for s in yo.SAMPLINGS), {s: len(v) for s, v in sizes.items()}
    for s in yo.SAMPLINGS:
        ws = {w for w, h in sizes[s]}
        assert (1, 1) in sizes[s] and any(w == 1 and h > 1 for w, h in sizes[s]) and any(h == 1 and w > 1 for w, h in sizes[s])
        if s != yo.S444:
            assert {(w + 1) // 2 for w in ws} >= {1, 2, 3}
    assert "preimage" in str(_Z["weak_422"])


def test_the_clamps_are_met():
    """the fixture's expected outputs reach 0 and 255, where the clamps decide"""
    lo = hi = 0
    for name in CASES:
        s, y, cb, cr, want = golden_case(name)
        lo += int((want[..., :3] == 0).sum())
        hi += int((want[..., :3] == 255).sum())
    assert lo > 100 and hi > 100


def test_hand_derived_values():
    """jdcolor.c's tables at a few points: neutral chroma is the identity; the extremes clamp"""
    y = np.array([[0, 128, 255]], np.uint8)
    n = np.full((1, 3), 128, np.uint8)
    assert yo.convert(yo.S444, y, n, n)[0, :, :3].tolist() == [[0, 0, 0], [128, 128, 128], [255, 255, 255]]
    px = yo.convert(yo.S444, np.array([[128]]), np.array([[255]]), np.array([[0]]))[0, 0]
    # cb - 128 = 127, cr - 128 = -128: R = 128 + ((91881 * -128 + 32768) >> 16) = -51 -> 0;
    # G = 128 + ((-22554 * 127 + 32768 + 46802 * 128) >> 16) = 176; B = 128 + ((116130 * 127 + 32768) >> 16) = 353 -> 255
    assert px.tolist() == [255, 176, 0, 255]


def test_upsampling_by_hand():
    """h2v1 and h2v2 at a three-column plane, and replication at a two-column one"""
    c = np.array([[0, 100, 200]])
    assert yo.upsample(yo.S422, c, 6, 1).tolist() == [[0, 25, 75, 125, 175, 200]]
    assert yo.upsample(yo.S422, c, 5, 1).tolist() == [[0, 25, 75, 125, 175]]
    assert yo.upsample(yo.S422, np.array([[0, 100]]), 4, 1).tolist() == [[0, 0, 100, 100]]
    c2 = np.array([[0, 100, 200], [40, 40, 40]])
    up = yo.upsample(yo.S420, c2, 6, 4)
    # row 0: s = 4 * row 0 (edge repeated) -> (0, 400, 800); column 1 = (3 * 0 + 400 + 7) >> 4 = 25
    assert up[0].tolist() == [0, 25, 75, 125, 175, 200]
    # row 1: s = 3 * row 0 + row 1 = (40, 340, 640); column 0 = (4 * 40 + 8) >> 4 = 10, column 1 = (120 + 340 + 7) >> 4 = 29
    assert up[1, :2].tolist() == [10, 29]
    assert yo.upsample(yo.S420, np.array([[0, 100], [40, 40]]), 3, 3).tolist() == [[0, 0, 100], [0, 0, 100], [40, 40, 40]]
