"""The CPU oracle of flow_bitmap_bgra_clear_around_rounded_corners (graphics/rounded_corners.rs:1-346) against a float32
transcription of the reference loop written here in numpy, byte for byte, and against known answers of the op."""
import math

import numpy as np
import pytest

import oracle
from tests import round_corners_oracle as rco

F = np.float32
PCT, PIX, CIRCLE, PCT_CUSTOM, PIX_CUSTOM = range(5)
NAN, INF = float("nan"), float("inf")


# ---------------------------------------------------------------------------------------------- the transcription
def _usize(f):                                   # `f32 as usize`: saturating, NaN -> 0
    f = float(f)
    return 0 if not f > 0 else (2 ** 64 - 1 if f >= 2.0 ** 64 else int(f))


def _clamp(v, lo, hi):                           # f32::clamp: NaN stays NaN
    if v < lo:
        v = lo
    if v > hi:
        v = hi
    return F(v)


def _fmax(a, b):
    return b if a != a else (a if b != b else max(a, b))


def _fmin(a, b):
    return b if a != a else (a if b != b else min(a, b))


def _plan(r, w, h):                              # plan_quadrants for Custom([tl, tr, bl, br]); (which, x, y, w, h, radius, cx, cy, top, left)
    rhw, bhh = w // 2, h // 2
    lhw, thh = w - rhw, h - bhh
    return [("TL", 0, 0, lhw, thh, r[0], r[0], r[0], True, True),
            ("TR", lhw, 0, rhw, thh, r[1], F(w) - r[1], r[1], True, False),
            ("BL", 0, thh, lhw, bhh, r[2], r[2], F(h) - r[2], False, True),
            ("BR", lhw, thh, rhw, bhh, r[3], F(w) - r[3], F(h) - r[3], False, False)]


def ref_round_corners(img, mode, radius, matte, t_lin, lut):
    """rounded_corners.rs:187-346 statement by statement, f32 scalars; img (h, w, 4) uint8 is modified.  Returns the mask of
    pixels written."""
    h, w = img.shape[:2]
    touched = np.zeros((h, w), np.uint8)
    if w == 0 or h == 0:
        return touched
    m = np.array(matte, np.uint8)
    a2f = F(1.0) / F(255.0)
    matte_a = F(int(matte[3])) * a2f
    mt = [t_lin[matte[0]], t_lin[matte[1]], t_lin[matte[2]]]
    vo = F(0.56419)
    smallest = F(min(w, h))
    tl, tr, br, bl = [F(v) for v in radius]
    if mode == CIRCLE:
        s = min(w, h)
        ox, oy = max(w - h, 0) // 2, max(h - w, 0) // 2
        v = smallest / F(2.0)
        quads = [(q[0], q[1] + ox, q[2] + oy, q[3], q[4], q[5], q[6] + F(ox), q[7] + F(oy), q[8], q[9]) for q in _plan([v] * 4, s, s)]
    else:
        pct = lambda p: smallest * _clamp(p, F(0), F(100)) / F(200)
        pix = lambda p: _clamp(p, F(0), smallest / F(2))
        if mode == PCT:
            r = [pct(tl)] * 4
        elif mode == PIX:
            r = [pix(tl)] * 4
        elif mode == PCT_CUSTOM:
            r = [pct(tl), pct(tr), pct(bl), pct(br)]
        else:
            r = [pix(tl), pix(tr), pix(bl), pix(br)]
        quads = _plan(r, w, h)

    def fill(x1, y1, x2, y2):
        img[y1:y2, x1:x2] = m
        touched[y1:y2, x1:x2] = 1

    for which, qx, qy, qw, qh, radius_, cx, cy, is_top, is_left in quads:
        bottom, right = qy + qh, qx + qw
        if qy > 0 and which == "TL":
            fill(0, 0, w, qy)
        if h > bottom and which == "BL":
            fill(0, bottom, w, h)
        rc = _usize(math.ceil(radius_)) if radius_ == radius_ else 0
        start_y = qy if is_top else bottom - rc
        end_y = qy + rc if is_top else bottom
        cf, ct = (0, qx) if is_left else (right, w)
        if cf != ct:
            for y in list(range(qy, start_y)) + list(range(end_y, bottom)):
                fill(cf, y, ct, y + 1)
        roi = radius_ + (F(1.0) - vo)
        ros = radius_ - vo
        raw = roi - ros
        roi2, ros2 = roi * roi, ros * ros
        for y in range(start_y, end_y):
            yf = F(y) + F(0.5)
            yd = abs(cy - yf)
            yd2 = yd * yd
            xds = np.sqrt(_fmax(ros2 - yd2, F(0)))
            xdi = np.sqrt(_fmax(roi2 - yd2, F(0)))
            es1 = _usize(_fmax(F(np.ceil(cx - xds)), F(0)))
            es2 = _usize(_fmin(F(np.floor(cx + xds)), F(w)))
            ei1 = _usize(_fmax(F(np.floor(cx - xdi)), F(0)))
            ei2 = _usize(_fmin(F(np.ceil(cx + xdi)), F(w)))
            if is_left:
                fill(0, y, ei1, y + 1)
            else:
                fill(ei2, y, w, y + 1)
            af, at = (ei1, es1) if is_left else (es2, ei2)
            for x in range(af, at):
                xf = F(x) + F(0.5)
                dxx = cx - xf
                dist = np.sqrt(dxx * dxx + yd2)
                if dist > roi:
                    fill(x, y, x + 1, y + 1)
                elif dist > ros:
                    inten = (dist - ros) / raw
                    p = img[y, x].copy()
                    pa = F(int(p[3])) * a2f * (F(1) - inten)
                    ma = (F(1) - pa) * matte_a
                    fa = ma + pa
                    out = []
                    for c in range(3):
                        with np.errstate(invalid="ignore", divide="ignore"):
                            lin = (t_lin[p[c]] * pa + mt[c] * ma) / fa
                        s = lin * F(16383)
                        out.append(lut[0 if not s > 0 else int(min(s, F(16383)))])
                    out.append(oracle.lib().ifo_uchar_clamp_ff(float(F(255) * fa)))
                    img[y, x] = out
                    touched[y, x] = 1
    return touched


@pytest.fixture(scope="module")
def tables():
    return oracle.byte_to_float_table(True), oracle.linear_to_srgb_table()


def _case(img, mode, radius, matte, tables):
    a = img.copy(); b = img.copy()
    want_mask = ref_round_corners(a, mode, radius, matte, *tables)
    got_mask = rco.round_corners(b, mode, radius, matte, want_mask=True)
    assert np.array_equal(a, b), (img.shape, mode, radius, matte, np.argwhere(np.any(a != b, axis=2))[:5])
    assert np.array_equal(want_mask, got_mask > 0), (img.shape, mode, radius)
    return b, got_mask


RADII = [0.0, 0.3, 1.0, 2.0, 2.5, 3.7, 7.0, 12.5, 19.5, 50.0, 150.0, -3.0, NAN, INF, -INF]


def _random_img(rng, h, w):
    img = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
    img[..., 3][rng.random((h, w)) < 0.2] = 0
    img[..., 3][rng.random((h, w)) < 0.3] = 255
    return img


def test_oracle_matches_transcription_every_small_size(tables):
    rng = np.random.default_rng(7)
    for h in range(1, 41):
        for w in range(1, 41):
            mode = int(rng.integers(0, 5))
            radius = tuple(float(rng.choice(RADII)) if rng.random() < 0.5 else float(rng.uniform(0, 25)) for _ in range(4))
            if mode in (PCT, PCT_CUSTOM) and rng.random() < 0.3:
                radius = tuple(float(rng.choice([0.0, 10.0, 33.3, 100.0, 140.0, 250.0])) for _ in range(4))
            matte = tuple(int(v) for v in rng.integers(0, 256, 4))
            if rng.random() < 0.2:
                matte = (0, 0, 0, 0)
            _case(_random_img(rng, h, w), mode, radius, matte, tables)


def test_oracle_matches_transcription_special_radii(tables):
    rng = np.random.default_rng(8)
    for r in RADII + [100.0, 101.0, 1e9]:
        for mode in range(5):
            for (h, w) in [(9, 9), (7, 12), (23, 16), (1, 5)]:
                radius = (r, r, r, r) if mode != PIX_CUSTOM else (r, 2.5, -1.0, NAN)
                _case(_random_img(rng, h, w), mode, radius, (12, 200, 90, int(rng.integers(0, 256))), tables)


def test_oracle_matches_transcription_large(tables):
    rng = np.random.default_rng(9)
    img = _random_img(rng, 400, 400)
    for mode, radius in [(PIX, (200.0,) * 4), (PCT, (37.5,) * 4), (CIRCLE, (0,) * 4), (PIX_CUSTOM, (50.0, 5.0, 100.0, 200.0))]:
        _case(img, mode, radius, (255, 0, 0, 255), tables)
    big = np.zeros((2160, 3840, 4), np.uint8); big[..., 1] = 180; big[..., 3] = 200
    _case(big, PIX, (100.0,) * 4, (0, 0, 0, 0), tables)
    _, mask = _case(big, CIRCLE, (0,) * 4, (10, 20, 30, 255), tables)
    assert mask[:, :840].all() and mask[:, 3000:].all() and not mask[1080, 1920]


# ---------------------------------------------------------------------------------------------- known answers
def test_outside_influence_is_matte_and_inside_solid_is_untouched():
    rng = np.random.default_rng(3)
    for (h, w, r) in [(60, 80, 20.0), (100, 30, 7.3), (50, 50, 12.5)]:        # corners that do not reach each other
        img = _random_img(rng, h, w)
        out = img.copy()
        matte = (1, 2, 3, 4)
        mask = rco.round_corners(out, PIX, (r,) * 4, matte, want_mask=True)
        roi, ros = r + (1 - 0.56419), r - 0.56419
        yc, xc = np.mgrid[0:h, 0:w] + 0.5
        d = np.hypot(xc - r, yc - r)                  # the top-left corner; the others are its mirror images
        tl = (xc <= r) & (yc <= r)
        for o, mk in [(out, mask), (out[:, ::-1], mask[:, ::-1]), (out[::-1], mask[::-1]), (out[::-1, ::-1], mask[::-1, ::-1])]:
            assert (o[tl & (d > roi + 1e-3)] == matte).all(), (h, w, r)
            assert not mk[tl & (d < ros - 1e-3)].any(), (h, w, r)
        rc = int(math.ceil(r))
        assert not mask[rc:h - rc].any() and not mask[:, rc:w - rc].any()
        ys, xs = np.nonzero(mask == 0)
        assert np.array_equal(out[ys, xs], img[ys, xs])


def test_transparent_pixel_under_transparent_matte_is_zero():
    img = np.zeros((30, 30, 4), np.uint8)
    img[..., :3] = 77                                   # colour under alpha 0
    out = img.copy()
    mask = rco.round_corners(out, PIX, (10.0,) * 4, (0, 0, 0, 0), want_mask=True)
    assert mask.any() and (out[mask == 1] == 0).all()


def test_overlapping_quadrants_equal_the_sequential_result(tables):
    rng = np.random.default_rng(5)
    # 5x5 at Pixels(2.5): the bottom quadrants' rows start one row above their quadrant; 100x99 with PixelsCustom 50/5/100/200
    for (h, w, mode, radius) in [(5, 5, PIX, (2.5,) * 4), (99, 100, PIX_CUSTOM, (50.0, 5.0, 100.0, 200.0))]:
        img = _random_img(rng, h, w)
        out, _ = _case(img, mode, radius, (0, 0, 0, 0xDD), tables)
        # not the same as applying each quadrant to the original image independently
        indep = img.copy()
        for keep in range(4):
            part = img.copy()
            rr = [radius[0]] * 4 if mode == PIX else list(radius)
            rr = [v if i == keep else 0.0 for i, v in enumerate(rr)]
            rco.round_corners(part, PIX_CUSTOM, rr, (0, 0, 0, 0xDD))
            changed = np.any(part != img, axis=2)
            indep[changed] = part[changed]
        assert not np.array_equal(indep, out)


def _hex_bgra(s):
    r, g, b, a = (int(s[i:i + 2], 16) for i in (0, 2, 4, 6))
    return (b, g, r, a)


# canvas.rs:239-388: CreateCanvas(w, h, Bgra32, colour) + RoundImageCorners(background_color, radius)
CANVAS_CASES = [
    ("test_round_corners_large", 400, 400, "FFFF00FF", "0000FFFF", PIX, (200.0,) * 4),
    ("test_round_corners_small", 100, 100, "FFFF00FF", "0000FFFF", PIX, (5.0,) * 4),
    ("test_round_corners_custom_pixels", 100, 99, "ddeecc88", "000000BB", PIX_CUSTOM, (0.0, 1.0, 50.0, 20.0)),
    ("test_round_corners_custom_percent", 100, 99, "2288ffEE", "000000DD", PIX_CUSTOM, (50.0, 5.0, 100.0, 200.0)),
    ("test_round_corners_excessive_radius", 200, 150, "FFFF00FF", "0000FFFF", PIX, (100.0,) * 4),
    ("test_round_corners_circle_wide_canvas", 200, 150, "FFFFFFFF", "000000FF", CIRCLE, (0.0,) * 4),
    ("test_round_corners_circle_tall_canvas", 150, 200, "FFFFFFFF", "00000000", CIRCLE, (0.0,) * 4),
]


@pytest.mark.parametrize("name,w,h,fill,matte,mode,radius", CANVAS_CASES, ids=[c[0] for c in CANVAS_CASES])
def test_reference_canvas_geometries(tables, name, w, h, fill, matte, mode, radius):
    img = np.empty((h, w, 4), np.uint8)
    img[...] = _hex_bgra(fill)
    m = _hex_bgra(matte)
    out, mask = _case(img, mode, radius, m, tables)
    assert tuple(out[0, 0]) == m and tuple(out[h - 1, w - 1]) == m or radius[0] == 0.0
    assert tuple(out[h // 2, w // 2]) == _hex_bgra(fill)
    if mode == CIRCLE:                                   # everything outside the centred square is the matte
        s = min(w, h); ox, oy = (w - s) // 2, (h - s) // 2
        assert (out[:oy] == m).all() and (out[oy + s:] == m).all() and (out[:, :ox] == m).all() and (out[:, ox + s:] == m).all()


def test_unknown_mode_is_an_error():
    with pytest.raises(oracle.OracleError):
        rco.round_corners(np.zeros((4, 4, 4), np.uint8), 5)
