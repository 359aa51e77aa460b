"""The closed form of include/ifb200.h against the reference's node expansions run node by node on the CPU oracle's flips and
transpose (tests/orient_oracle.py), for every flag and node kind on odd, non-square sizes; orientation_of against every chain of up
to three nodes; and RIAPI's rotate / flip steps against hand-derived cases.  No GPU is needed."""
import itertools

import numpy as np
import pytest

import imageflow_b200 as ifb
from tests import orient_oracle as oo

SIZES = [(1, 1), (1, 7), (7, 1), (5, 3), (33, 31)]
KINDS = [("ApplyOrientation", f) for f in range(-1, 10)] + list(oo.NODES)
PRODUCT_NODE = {oo.ROTATE_90: ifb.Rotate90, oo.ROTATE_180: ifb.Rotate180, oo.ROTATE_270: ifb.Rotate270, oo.FLIP_H: ifb.FlipH,
                oo.FLIP_V: ifb.FlipV, oo.TRANSPOSE: ifb.Transpose}


def _product_steps(steps):
    return [ifb.ApplyOrientation(s[1]) if isinstance(s, tuple) else PRODUCT_NODE[s] for s in steps]


def _noise(w, h, seed):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 4), dtype=np.uint8)


def test_the_table_is_what_the_expansions_do():
    """The table read off the expansions: run each flag's nodes on an image whose pixels carry their own coordinates, and the
    output pixel (x, y) names the input pixel it came from."""
    w, h = 5, 3
    derived = {}
    for f in range(1, 9):
        out = oo.run_nodes(oo.coordinate_image(w, h), [("ApplyOrientation", f)])
        sx, sy = oo.coordinates(out)
        oh, ow = out.shape[:2]
        y, x = np.indices((oh, ow))
        # each source coordinate is x, y, or their reversal w-1-.. / h-1-..; find which
        def name(s, label, n):
            for lab, v in (("x", x), ("y", y), (f"{label}-1-x", n - 1 - x), (f"{label}-1-y", n - 1 - y)):
                if np.array_equal(s, v):
                    return lab
        derived[f] = (name(sx, "w", w), name(sy, "h", h))
    assert derived == {1: ("x", "y"), 2: ("w-1-x", "y"), 3: ("w-1-x", "h-1-y"), 4: ("x", "h-1-y"), 5: ("y", "x"), 6: ("y", "h-1-x"),
                       7: ("w-1-y", "h-1-x"), 8: ("w-1-y", "x")}


@pytest.mark.parametrize("w,h", SIZES)
@pytest.mark.parametrize("kind", KINDS, ids=[k if isinstance(k, str) else f"ApplyOrientation({k[1]})" for k in KINDS])
def test_each_node_kind_is_its_orientations_gather(kind, w, h):
    img = _noise(w, h, w * 100 + h)
    want = oo.run_nodes(img, [kind])
    o = ifb.orientation_of(_product_steps([kind]))
    assert np.array_equal(oo.gather(img, o), want)
    if isinstance(kind, tuple):
        assert o == (kind[1] if 2 <= kind[1] <= 8 else 1)


def test_every_chain_of_up_to_three_nodes_is_one_orientation():
    img = _noise(5, 3, 7)
    chains = [()] + [c for n in (1, 2, 3) for c in itertools.product(KINDS, repeat=n)]
    seen = set()
    for chain in chains:
        want = oo.run_nodes(img, chain)
        o = ifb.orientation_of(_product_steps(chain))
        assert np.array_equal(oo.gather(img, o), want), chain
        seen.add(o)
    assert seen == set(range(1, 9))


def test_riapi_rotate_steps_follow_rusts_integer_arithmetic():
    # add_rotate: match ((rot / 90) + 4) % 4 { 1 => Rotate90, 2 => Rotate180, 3 => Rotate270, _ => nothing }, i32 `/` and `%`
    cases = {0: [], 90: [ifb.Rotate90], 180: [ifb.Rotate180], 270: [ifb.Rotate270], 360: [], 450: [ifb.Rotate90],
             -90: [ifb.Rotate270], -180: [ifb.Rotate180], -270: [ifb.Rotate90], -360: [],
             45: [], 89: [], 135: [ifb.Rotate90], -45: [], -135: [ifb.Rotate270],
             -450: [],                   # -5 + 4 = -1, and -1 % 4 == -1 matches no arm
             -540: [], -630: [], -720: [], -810: [], 720: [], 810: [ifb.Rotate90]}    # from -450 down, (q + 4) % 4 is 0 or negative: no rotation
    for deg, want in cases.items():
        assert ifb.riapi_rotate_steps(deg) == want, deg


def test_riapi_flip_steps():
    assert ifb.riapi_flip_steps(False, False) == []
    assert ifb.riapi_flip_steps(True, False) == [ifb.FlipH]
    assert ifb.riapi_flip_steps(False, True) == [ifb.FlipV]
    assert ifb.riapi_flip_steps(True, True) == [ifb.FlipH, ifb.FlipV]


def test_autorotate_srotate_sflip_is_one_orientation():
    """ApplyOrientation(6), then srotate=90, then sflip=h: one flag that equals the node-by-node chain"""
    steps = [ifb.ApplyOrientation(6)] + ifb.riapi_rotate_steps(90) + ifb.riapi_flip_steps(True, False)
    o = ifb.orientation_of(steps)
    img = _noise(33, 31, 3)
    assert np.array_equal(oo.gather(img, o), oo.run_nodes(img, [("ApplyOrientation", 6), oo.ROTATE_90, oo.FLIP_H]))
    assert o == 4                                   # Rotate90 twice is Rotate180; with FlipH that leaves FlipV


def test_unknown_nodes_are_rejected():
    with pytest.raises(ifb.FlowError):
        ifb.orientation_of(["Rotate45"])
