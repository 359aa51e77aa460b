"""The argument behind ifb200_batch_watermark, made on the CPU: a watermark's resample F (oracle.resample_stages) composited over a
canvas with the store epilogue alone (tests/watermark_oracle.composite) equals oracle.scale_and_render byte for byte -- over several
different canvases from ONE F, through every compose mode, both watermark formats and both working spaces, on cut-out and noise
watermarks.  And the whole node (crop, Alpha, draw under the Compose rule) computed through one F per watermark equals the node-by-node
expansion."""
import numpy as np
import pytest

import imageflow_b200 as ifb
import oracle
from imageflow_b200 import synth
from tests import watermark_oracle as wo


def _wm(kind, w, h, seed):
    return synth.cutout_np(w, h, seed) if kind == "cutout" else synth.noise_np(w, h, seed, alpha_mode="mixed")


@pytest.mark.parametrize("kind", ["cutout", "noise"])
@pytest.mark.parametrize("linear", [True, False])
@pytest.mark.parametrize("am", [True, False])
@pytest.mark.parametrize("compose", [0, 1, 2])
def test_one_f_composited_over_many_canvases_equals_scale_and_render(kind, linear, am, compose):
    wm = _wm(kind, 97, 61, 3)
    for (w, h, filt) in ((40, 25, 2), (150, 90, 4)):
        f = wo.f_of(wm, am, w, h, filt, linear)
        for seed in range(3):
            cv = synth.cutout_canvas_np(w + 7, h + 5, seed) if seed != 1 else synth.noise_np(w + 7, h + 5, seed, alpha_mode="mixed")
            matte = (30, 200, 90, 140 + seed)
            exp = cv.copy()
            oracle.scale_and_render(wm, exp, x=3, y=2, w=w, h=h, filter=filt, linear=linear, alpha_meaningful=am, compose=compose, matte=matte)
            got = cv.copy()
            got[2:2 + h, 3:3 + w] = wo.composite(f, cv[2:2 + h, 3:3 + w], linear=linear, am=am, compose=compose, matte=matte)
            assert np.array_equal(got, exp), (w, h, seed, np.argwhere(got != exp)[:3].tolist())


@pytest.mark.parametrize("opacity", [None, 0.9, 0.3, 0.0])
@pytest.mark.parametrize("wm_am", [True, False])
@pytest.mark.parametrize("compose", [0, 1, 2])
def test_the_node_through_one_f_equals_the_node_by_node_expansion(opacity, wm_am, compose):
    wm = synth.cutout_np(120, 50, 7)
    spec = ifb.Watermark(fit_box=ifb.WatermarkConstraintBox.image_percentage(10, 20, 90, 95), fit_mode=ifb.WatermarkConstraintMode.FitCrop,
                         gravity=ifb.ConstraintGravity.percentage(30, 80), opacity=opacity)
    frames = [synth.cutout_canvas_np(160, 120, s) for s in range(3)]
    draw = ifb.watermark_layout(160, 120, 120, 50, spec)
    assert draw is not None and draw.crop is not None and (draw.opacity is None) == (opacity is None)
    src, am = wo.source_of(wm, wm_am, draw)
    f = wo.f_of(src, am, draw.w, draw.h, int(draw.filter))
    matte = (10, 20, 250, 200)
    for fr in frames:
        exp = fr.copy()
        wo.expansion(exp, compose, matte, wm, wm_am, draw)
        got = fr.copy()
        rect = (slice(draw.y, draw.y + draw.h), slice(draw.x, draw.x + draw.w))
        got[rect] = wo.composite(f, fr[rect], linear=True, am=am, compose=wo.drawn_compose(compose), matte=matte)
        assert np.array_equal(got, exp)
