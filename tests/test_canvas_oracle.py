"""The numpy oracle of the canvas operations (tests/canvas_oracle.py) against answers derived by hand from the reference source, and
the graphs of the reference's canvas visual tests (imageflow_core/tests/integration/visuals/canvas.rs) without their resample.  The
reference stores those graphs' results as seahash digests, which cannot be reproduced here; these tests check the pixel content each
graph's steps define instead."""
import numpy as np
import pytest

from tests import canvas_oracle as co


def _canvas(w, h, color, am=True):
    a = np.empty((h, w, 4), np.uint8)
    win = co.Win.of(a, am)
    co.create_canvas(win, color)
    return a, win


def test_hex_colours_are_to_bgra8_bytes():
    assert co.hex_bgra("EECCFFFF") == (0xFF, 0xCC, 0xEE, 0xFF)
    assert co.hex_bgra("FF0000") == (0, 0, 255, 255)
    assert co.hex_bgra("2233AA00") == (0xAA, 0x33, 0x22, 0)


def test_alpha_zero_colour_fills_its_own_bytes():
    a, win = _canvas(5, 4, co.hex_bgra("2233AA00"))
    assert (a == (0xAA, 0x33, 0x22, 0)).all()
    co.fill_rectangle(win, (9, 8, 7, 0), 1, 1, 3, 2)
    assert tuple(a[1, 1]) == (9, 8, 7, 0) and tuple(a[1, 3]) == (0xAA, 0x33, 0x22, 0)


def test_zero_size_fill_out_of_bounds_is_a_no_op():
    a, win = _canvas(4, 4, (1, 2, 3, 4))
    before = a.copy()
    for r in [(10, 10, 10, 20), (7, 3, 9, 3), (0, 0, 0, 0)]:
        co.fill_rectangle(win, (9, 9, 9, 9), *r)
    assert np.array_equal(a, before)
    for r in [(0, 0, 5, 1), (0, 0, 1, 5), (2, 0, 1, 1), (0, 2, 1, 1)]:
        with pytest.raises(co.CanvasArgError):
            co.fill_rectangle(win, (9, 9, 9, 9), *r)


def test_bgr32_input_into_bgra32_canvas():
    """ExpandCanvas with a colour that is not opaque: a Bgra32 canvas; the Bgr32 input's whole window gets A = 255 in place"""
    inp = np.full((3, 4, 4), 7, np.uint8)
    inp[..., 3] = np.arange(12).reshape(3, 4)
    iw = co.Win.of(inp, False)
    out = np.empty((5, 7, 4), np.uint8)
    cv = co.Win.of(out)
    co.expand_canvas(iw, cv, 1, 1, 2, 1, (10, 20, 30, 40))
    assert cv.alpha_meaningful and not iw.alpha_meaningful
    assert (out[1:4, 1:5] == (7, 7, 7, 255)).all()
    assert (inp[..., 3] == 255).all()
    border = np.ones((5, 7), bool); border[1:4, 1:5] = False
    assert (out[border] == (10, 20, 30, 40)).all()


def test_bgr32_canvas_under_bgra32_input():
    cv_px = np.full((4, 6, 4), 3, np.uint8)
    cv = co.Win.of(cv_px, False)
    src = np.full((2, 2, 4), 9, np.uint8)
    co.copy_rectangle(co.Win.of(src, True), cv, 0, 0, 4, 2, 2, 2)
    assert cv.alpha_meaningful
    assert (cv_px[..., 3][:, :4] == 255).all() and (cv_px[:2, :4, :3] == 3).all()
    assert (cv_px[2:, 4:] == 9).all()                          # the copy is raw: the input's alpha 9 stays
    assert (src == 9).all()


def test_opaque_expand_keeps_the_input_format_and_copies_raw_bytes():
    inp = np.full((2, 2, 4), 5, np.uint8)
    out = np.empty((4, 4, 4), np.uint8)
    cv = co.Win.of(out)
    co.expand_canvas(co.Win.of(inp, False), cv, 1, 1, 1, 1, (1, 2, 3, 255))
    assert not cv.alpha_meaningful and (out[1:3, 1:3] == 5).all() and (inp == 5).all()


def test_zero_size_copy_is_an_error():
    a = np.zeros((4, 4, 4), np.uint8)
    with pytest.raises(co.CanvasArgError):
        co.copy_rectangle(co.Win.of(a.copy()), co.Win.of(a), 0, 0, 0, 0, 0, 2)


def test_red_dot():
    assert co.watermark_red_dot(3, 3) is None and co.watermark_red_dot(4, 3) is None
    a, win = _canvas(4, 4, (1, 1, 1, 1))
    x1, y1, x2, y2, c = co.watermark_red_dot(4, 4)
    co.fill_rectangle(win, c, x1, y1, x2, y2)
    assert (x1, y1, x2, y2) == (1, 1, 4, 4) and (a[1:, 1:] == (0, 0, 255, 255)).all() and (a[0] == 1).all() and (a[:, 0] == 1).all()


# ------------------------------------------------------------------------------------------------ canvas.rs graphs
RED, BLUE = co.hex_bgra("FF5555FF"), co.hex_bgra("0000FFFF")


def _red_with_blue_strip():
    a, win = _canvas(200, 200, RED)
    co.fill_rectangle(win, BLUE, 0, 0, 10, 100)
    return a


def test_fill_rect_original():
    a, win = _canvas(400, 300, co.TRANSPARENT)
    co.fill_rectangle(win, BLUE, 0, 0, 50, 100)
    assert (a[:100, :50] == BLUE).all() and (a[100:] == 0).all() and (a[:, 50:] == 0).all()


def test_crop():
    a = _red_with_blue_strip()
    crop = co.Win.of(a, True).sub(0, 50, 100, 100).px()
    assert crop.shape == (50, 100, 4) and (crop[:, :10] == BLUE).all() and (crop[:, 10:] == RED).all()


def test_transparent_canvas():
    a, _ = _canvas(200, 200, co.hex_bgra("00000000"))
    assert (a == 0).all()


def test_off_surface_region():
    coords = co.region_percent_coords(200, 200, -100.0, -100.0, -1.0, -1.0)
    assert coords == (-200, -200, -2, -2)
    out, am = co.run_region(_red_with_blue_strip(), True, *coords, co.TRANSPARENT)
    assert out.shape == (198, 198, 4) and (out == 0).all() and am


def test_partial_region():
    coords = co.region_percent_coords(200, 200, -10.0, -10.0, 40.0, 40.0)
    assert coords == (-20, -20, 80, 80)
    out, am = co.run_region(_red_with_blue_strip(), True, *coords, co.TRANSPARENT)
    assert out.shape == (100, 100, 4) and am
    assert (out[:20] == 0).all() and (out[:, :20] == 0).all()
    assert (out[20:, 20:30] == BLUE).all() and (out[20:, 30:] == RED).all()


def test_pixels_region():
    out, am = co.run_region(_red_with_blue_strip(), True, -10, -10, 120, 50, co.TRANSPARENT)
    assert out.shape == (60, 130, 4)
    assert (out[:10] == 0).all() and (out[:, :10] == 0).all()
    assert (out[10:, 10:20] == BLUE).all() and (out[10:, 20:] == RED).all()


def test_expand_rect_without_its_resample():
    a, win = _canvas(200, 200, co.TRANSPARENT)
    co.fill_rectangle(win, co.hex_bgra("EECCFFFF"), 0, 0, 100, 100)
    out = np.empty((240, 230, 4), np.uint8)
    cv = co.Win.of(out)
    co.expand_canvas(win, cv, 10, 15, 20, 25, co.hex_bgra("2233AAFF"))
    assert cv.alpha_meaningful
    inner = out[15:215, 10:210]
    assert np.array_equal(inner, a)
    assert (inner[:100, :100] == (0xFF, 0xCC, 0xEE, 0xFF)).all() and (inner[100:] == 0).all()
    border = np.ones((240, 230), bool); border[15:215, 10:210] = False
    assert (out[border] == (0xAA, 0x33, 0x22, 0xFF)).all()


def test_region_percent_rounds_halves_away_from_zero():
    assert co.region_percent_coords(5, 5, 10.0, 10.0, 50.0, 50.0) == (1, 1, 3, 3)     # 0.5 -> 1, 2.5 -> 3
    assert co.region_percent_coords(5, 5, -10.0, -10.0, 50.0, 50.0)[:2] == (-1, -1)
