"""CropWhitespace's arithmetic in the mirror (imageflow_b200.crop_whitespace_bounds; clone_crop_fill_expand.rs:585-605 and the check
of Bitmap::crop, bitmaps.rs:841-851) against a numpy f32 restatement, and riapi_trim_steps (ir4/mod.rs:107-111).  No GPU."""
import numpy as np
import pytest

import imageflow_b200 as ifb

I64 = 2**63


def reference(rect, w, h, p):
    """the node's arithmetic restated: f32 padding, Rust's saturating f32 -> i64, wrapping i64 sums, `as u32`"""
    x1, y1, x2, y2 = rect
    if x2 <= x1 or y2 <= y1:
        return "InvalidState"
    with np.errstate(all="ignore"):
        f = np.ceil(np.float32(p) / np.float32(100) * np.float32(x2 - x1 + y2 - y1) / np.float32(2)).astype(np.float32)
    pad = 0 if np.isnan(f) else (I64 - 1 if f >= 2.0**63 else -I64 if f <= -2.0**63 else int(f))
    wrap = lambda v: (v + I64) % 2**64 - I64
    c = (max(0, wrap(x1 - pad)) % 2**32, max(0, wrap(y1 - pad)) % 2**32, min(w, wrap(x2 + pad)) % 2**32, min(h, wrap(y2 + pad)) % 2**32)
    if c[2] <= c[0] or c[3] <= c[1] or c[2] > w or c[3] > h:
        return "InvalidArgument"
    return c


PERCENTS = [0.0, 0.02, 0.5, 10.0, -30.0, 1e30, -1e30, float("nan"), float("inf")]


def test_padding_and_crop_match_the_restatement():
    rng = np.random.default_rng(7)
    cases = [((80, 80, 120, 120), 200, 200), ((0, 0, 1, 1), 1, 1), ((59, 0, 59, 49), 60, 50), ((3, 4, 3000, 1999), 4000, 2000),
             ((100, 100, 200, 200), 300, 300), ((0, 0, 4000, 3000), 4000, 3000)]
    for _ in range(300):
        w, h = int(rng.integers(1, 5000)), int(rng.integers(1, 5000))
        x1, x2 = sorted(int(v) for v in rng.integers(0, w + 1, 2)); y1, y2 = sorted(int(v) for v in rng.integers(0, h + 1, 2))
        cases.append(((x1, y1, x2, y2), w, h))
    for rect, w, h in cases:
        for p in PERCENTS + [float(rng.uniform(-60, 60))]:
            want = reference(rect, w, h, p)
            if isinstance(want, str):
                with pytest.raises(ifb.FlowError) as e:
                    ifb.crop_whitespace_bounds(rect, w, h, p)
                assert e.value.kind == ifb.ErrorKind[want], (rect, w, h, p)
            else:
                assert ifb.crop_whitespace_bounds(rect, w, h, p) == want, (rect, w, h, p)


def test_known_answers():
    assert ifb.crop_whitespace_bounds((80, 80, 120, 120), 200, 200, 10.0) == (76, 76, 124, 124)     # ceil(0.1 * 80 / 2) = 4
    assert ifb.crop_whitespace_bounds((80, 80, 120, 120), 200, 200, 0.02) == (79, 79, 121, 121)     # ceil(0.008) = 1
    assert ifb.crop_whitespace_bounds((80, 80, 120, 120), 200, 200, float("nan")) == (80, 80, 120, 120)
    # 1e30 % saturates to i64::MAX: x1 - pad clamps to 0, x2 + pad wraps (a release build's i64 add) and `as u32` keeps x2 - 1
    assert ifb.crop_whitespace_bounds((80, 80, 120, 120), 200, 200, 1e30) == (0, 0, 119, 119)
    with pytest.raises(ifb.FlowError, match="Invalid crop bounds") as e:
        ifb.crop_whitespace_bounds((80, 80, 120, 120), 200, 200, -60.0)
    assert e.value.kind == ifb.ErrorKind.InvalidArgument
    with pytest.raises(ifb.FlowError, match="Whitespace detection returned invalid rectangle") as e:     # the last-column frame
        ifb.crop_whitespace_bounds((59, 0, 59, 49), 60, 50, 0.0)
    assert e.value.kind == ifb.ErrorKind.InvalidState


def test_riapi_trim_steps():
    assert ifb.riapi_trim_steps() == [] and ifb.riapi_trim_steps(None, 5) == []
    assert ifb.riapi_trim_steps(80) == [ifb.CropWhitespace(80, 0.0)]
    assert ifb.riapi_trim_steps(-5, 0.5) == [ifb.CropWhitespace(0, float(np.float32(0.5)))]
    assert ifb.riapi_trim_steps(20, 10) == [ifb.CropWhitespace(20, 10.0)]
