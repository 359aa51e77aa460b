"""The Python mirror of the Watermark node's layout (imageflow_b200.graphics: process_constraint, watermark_layout,
riapi_watermark_placement) against hand-derived answers for the five watermark modes, the reference's own sizing answers
(tests/golden/watermark_sizing.json), half-way roundings where f32 and Rust's rounding matter, the cases where the node deletes itself,
the opacity rule and the RIAPI placement.  No GPU is needed."""
import json
import math
import os

import numpy as np
import pytest

import imageflow_b200 as ifb
from imageflow_b200 import graphics as g

M, B, G = ifb.WatermarkConstraintMode, ifb.WatermarkConstraintBox, ifb.ConstraintGravity
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "watermark_sizing.json")


def test_the_reference_sizing_answers():
    data = json.load(open(GOLDEN))
    for c in data["box_of"]:
        r = g._Ratio(*c["ratio"]).box_of(g._Ratio(*c["target"]), c["kind"] == "inner")
        assert [r.w, r.h] == c["expect"], c
    for c in data["process_constraint"]:
        crop, scale_to = ifb.process_constraint(*c["src"], M[c["mode"]], *c["box"])
        assert list(scale_to) == c["scale_to"], c
        assert (None if crop is None else [crop[2] - crop[0], crop[3] - crop[1]]) == c["crop_size"], c


@pytest.mark.parametrize("mode, src, box, gravity, crop, scale_to", [
    # Distort: exactly the box, never a crop
    (M.Distort, (400, 100), (60, 90), None, None, (60, 90)),
    (M.Distort, (100, 400), (600, 900), None, None, (600, 900)),
    # Within: only scales down, inside the box; a smaller watermark keeps its size
    (M.Within, (400, 100), (200, 200), None, None, (200, 50)),
    (M.Within, (100, 400), (200, 200), None, None, (50, 200)),
    (M.Within, (40, 10), (200, 200), None, None, (40, 10)),
    # Fit: scales up too
    (M.Fit, (40, 10), (200, 200), None, None, (200, 50)),
    (M.Fit, (10, 40), (200, 300), None, None, (75, 300)),
    (M.Fit, (400, 100), (200, 200), None, None, (200, 50)),
    (M.Fit, (100, 400), (200, 200), None, None, (50, 200)),
    # FitCrop: fills the box, crops the overflow at the gravity (centre: round((400 - 100) * 0.5) = 150; 100 %: 300; 0 %: 0)
    (M.FitCrop, (400, 100), (100, 100), None, [150, 0, 250, 100], (100, 100)),
    (M.FitCrop, (400, 100), (100, 100), G.percentage(100, 0), [300, 0, 400, 100], (100, 100)),
    (M.FitCrop, (100, 400), (50, 100), G.percentage(0, 25), [0, 50, 100, 250], (50, 100)),
    (M.FitCrop, (40, 10), (300, 300), None, [15, 0, 25, 10], (300, 300)),
    # WithinCrop: larger in both -> scale to the outer box and crop; smaller in one dimension -> crop to the intersection, no scale
    (M.WithinCrop, (400, 100), (100, 50), None, [100, 0, 300, 100], (100, 50)),
    (M.WithinCrop, (400, 100), (100, 200), G.percentage(100, 100), [300, 0, 400, 100], (100, 100)),
    (M.WithinCrop, (40, 10), (100, 200), None, None, (40, 10)),
    (M.WithinCrop, (100, 400), (50, 100), None, [0, 100, 100, 300], (50, 100)),
    (M.WithinCrop, (100, 40), (50, 100), None, [25, 0, 75, 40], (50, 40)),
    (M.WithinCrop, (40, 100), (100, 50), None, [0, 25, 40, 75], (40, 50)),
    (M.WithinCrop, (40, 100), (100, 50), G.percentage(0, 100), [0, 50, 40, 100], (40, 50)),
])
def test_hand_derived_answers_for_the_five_modes(mode, src, box, gravity, crop, scale_to):
    got_crop, got_scale = ifb.process_constraint(*src, mode, *box, gravity)
    assert got_crop == crop and tuple(got_scale) == scale_to


def test_f32_half_way_roundings():
    # ImagePercentage 50 % of 101 = 50.5 in f32 -> 51 (half away from zero; Python's round gives 50)
    d = ifb.watermark_layout(101, 101, 10, 10, ifb.Watermark(fit_box=B.image_percentage(50, 50, 100, 100), gravity=G.percentage(0, 0)))
    assert (d.x, d.y) == (51, 51) and round(50.5) == 50
    # gravity 50 % of (61 - 10) = 25.5 -> 26; 12.5 % of 20 = 2.5 -> 3
    d = ifb.watermark_layout(61, 30, 10, 10, ifb.Watermark())
    assert d.x == 26 and d.y == 10
    d = ifb.watermark_layout(30, 30, 10, 10, ifb.Watermark(gravity=G.percentage(12.5, 12.5)))
    assert (d.x, d.y) == (3, 3)
    # 0.1 is not exact in f32: 33.3 % of 1000 = 333.0 (f32: 0.333 * 1000 = 332.99997 -> 333)
    assert g._fit_box(1000, 1000, B.image_percentage(33.3, 0, 100, 100))[0] == int(np.round(np.float32(33.3) / np.float32(100) * np.float32(1000)))


def test_gravity_of_the_node_is_not_clamped_but_the_layouts_is():
    assert g._wm_gravity1d(100.0, 30, 20) == -10                # the watermark is larger than the box: no clamp
    assert g._ir4_gravity1d(100.0, 30, 20) == 0
    with pytest.raises(ifb.FlowError) as e:
        g._wm_gravity1d(50.0, 5, 0)
    assert e.value.kind == ifb.ErrorKind.InvalidNodeParams


def test_min_canvas_equal_to_the_frame_deletes_the_node():
    assert ifb.watermark_layout(200, 100, 10, 10, ifb.Watermark(min_canvas_width=200)) is None
    assert ifb.watermark_layout(200, 100, 10, 10, ifb.Watermark(min_canvas_height=100)) is None
    assert ifb.watermark_layout(200, 100, 10, 10, ifb.Watermark(min_canvas_width=199, min_canvas_height=99)) is not None


def test_a_fit_box_too_small_deletes_the_node():
    assert ifb.watermark_layout(200, 100, 10, 10, ifb.Watermark(fit_box=B.image_margins(100, 0, 100, 0))) is None
    assert ifb.watermark_layout(200, 100, 10, 10, ifb.Watermark(fit_box=B.canvas_percentage(50, 0, 50.2, 100))) is None
    assert ifb.watermark_layout(200, 100, 10, 10, ifb.Watermark(fit_box=B.canvas_percentage(50, 0, 50.3, 100))) is not None


@pytest.mark.parametrize("opacity, applied", [(None, None), (float("nan"), None), (-0.5, 0.0), (0.0, 0.0), (0.3, np.float32(0.3)),
                                              (1.0, None), (7.0, None)])
def test_the_opacity_rule(opacity, applied):
    d = ifb.watermark_layout(100, 100, 10, 10, ifb.Watermark(opacity=opacity))
    assert d.opacity == (None if applied is None else float(applied))


def test_hints_with_another_filter_give_the_same_draw():
    base = ifb.Watermark(fit_mode=M.Fit)
    hinted = ifb.Watermark(fit_mode=M.Fit, hints={"down_filter": "Lanczos", "up_filter": "Mitchell", "sharpen_percent": 15})
    for (fw, fh, ww, wh) in ((300, 200, 40, 40), (300, 200, 900, 100)):
        assert ifb.watermark_layout(fw, fh, ww, wh, base) == ifb.watermark_layout(fw, fh, ww, wh, hinted)
    assert ifb.watermark_layout(300, 200, 40, 40, base).filter == ifb.Filter.Ginseng          # up-scale
    assert ifb.watermark_layout(300, 200, 900, 100, base).filter == ifb.Filter.Robidoux       # down-scale


def test_before_and_after_pad_placement():
    ws = [ifb.Watermark(io_id=1, fit_box=B.canvas_margins(1, 1, 1, 1)), ifb.Watermark(io_id=2), ifb.Watermark(io_id=3, fit_box=B.image_percentage(0, 0, 1, 1)),
          ifb.Watermark(io_id=4, fit_box=B.canvas_percentage(0, 0, 1, 1)), ifb.Watermark(io_id=5, fit_box=B.image_margins(0, 0, 0, 0))]
    before, after = ifb.riapi_watermark_placement(ws)
    assert [w.io_id for w in before] == [2, 3, 5] and [w.io_id for w in after] == [1, 4]
    assert ifb.riapi_watermark_placement(None) == ([], [])
