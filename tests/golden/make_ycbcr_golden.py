"""python tests/golden/make_ycbcr_golden.py: writes tests/golden/ycbcr_golden.npz, libjpeg-turbo's decoder colour stage (upsampling and
YCbCr -> RGB) on raw Y, Cb and Cr planes, with Pillow's bundled libjpeg-turbo as the decoder.  Needs Pillow; the tests read only the
.npz.

For each seeded image and sampling, the image is encoded as a baseline JPEG and decoded three ways:
  - full scale as "YCbCr" (out_color_space = JCS_YCbCr): Y, and the chroma upsampled as the RGB decode upsamples it;
  - full scale as "RGB": the expected output, stored as BGRA with alpha 255 (what JCS_EXT_BGRA writes);
  - for 4:2:0, at DCT scale 1/2 as "YCbCr": libjpeg-turbo then scales the luma IDCT to 4x4 and leaves the chroma at 8x8, so the Cb and
    Cr planes come out at their stored resolution -- the raw chroma a GPU decoder hands over.
Raw planes per sampling:
  4:4:4  the full-scale YCbCr decode.
  4:2:0  Y from the full-scale decode; Cb and Cr from the half-scale decode, checked by upsampling them (tests/ycbcr_oracle.py) and
         comparing with the full-scale decode's chroma.
  4:2:2  Pillow gives no raw 4:2:2 chroma, so each chroma row is solved for: a row whose h2v1 upsampling reproduces the full-scale
         decode's row (a search over each sample's candidates, left to right).  This pins 4:2:2 more weakly than the other two
         samplings: the planes are a preimage of libjpeg-turbo's upsampling, not the planes its IDCT produced ("weak_422" in the file).
Cases whose preimage search fails are not written (none at the seeds below)."""
import io
import os

import numpy as np
from PIL import Image, ImageFile, features

import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from tests import ycbcr_oracle as yo  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ycbcr_golden.npz")
SIZES = [(1, 1), (2, 2), (1, 9), (13, 1), (2, 7), (3, 3), (4, 5), (5, 3), (6, 2), (7, 11), (8, 8), (9, 16), (16, 9), (17, 17),
         (31, 6), (37, 23), (64, 48), (101, 7), (7, 101), (128, 96), (250, 33)]
PIL_SUBSAMPLING = {yo.S444: 0, yo.S422: 1, yo.S420: 2}


def image(w, h, seed):
    """a seeded image with smooth colour and noise, so that both flat chroma and the clamps are met"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([128 + 120 * np.sin(xx / 5.0 + c + seed) * np.cos(yy / 7.0 - c) for c in range(3)], axis=-1)
    return np.clip(base + rng.normal(0, 40, (h, w, 3)), 0, 255).astype(np.uint8)


def decode(data, mode, half=False):
    im = Image.open(io.BytesIO(data))
    if half:                                        # Image.draft at scale 1/2 for every size (draft itself needs w, h >= 2)
        d, e, o, a = im.tile[0]
        im._mode = mode
        im.tile = [ImageFile._Tile(d, (e[0], e[1], (e[2] + 1) // 2, (e[3] + 1) // 2), o, (mode, ""))]
        im._size = ((im.size[0] + 1) // 2, (im.size[1] + 1) // 2)
        im.decoderconfig = (2, 0)
    else:
        im = im.convert(mode) if mode == "RGB" else im
        if mode == "YCbCr":
            im.draft("YCbCr", None)
    return np.asarray(im)


def solve_h2v1(row, n):
    """a chroma row of n samples whose h2v1 upsampling equals `row` (len w), or None"""
    w = row.shape[0]
    if n <= 2:
        return row[0::2].astype(np.uint8)           # replicated: the samples are the even columns
    # depth-first over samples left to right; each sample is pinned by the output columns it alone decides
    out = np.zeros(n, np.int64)

    def ok_prefix(k):
        c = out[:k + 1]
        for x in range(min(w, 2 * k + 2)):
            i = x // 2
            nb = i - 1 if x % 2 == 0 else i + 1
            nb = min(max(nb, 0), n - 1)
            if nb > k:
                continue
            v = (3 * c[i] + c[nb] + (1 if x % 2 == 0 else 2)) >> 2
            if v != row[x]:
                return False
        return True

    def rec(k):
        if k == n:
            return True
        for v in np.argsort(np.abs(np.arange(256) - int(row[min(2 * k, w - 1)])), kind="stable"):
            out[k] = v
            if ok_prefix(k) and rec(k + 1):
                return True
        return False

    sys.setrecursionlimit(10000)
    return out.astype(np.uint8) if rec(0) else None


def case(w, h, sampling, seed):
    buf = io.BytesIO()
    Image.fromarray(image(w, h, seed)).save(buf, "JPEG", quality=88, subsampling=PIL_SUBSAMPLING[sampling])
    data = buf.getvalue()
    full = decode(data, "YCbCr")
    rgb = decode(data, "RGB")
    assert full.shape == (h, w, 3) and rgb.shape == (h, w, 3)
    y = full[..., 0].copy()
    ch, cw = yo.chroma_shape(sampling, w, h)
    if sampling == yo.S444:
        cb, cr = full[..., 1].copy(), full[..., 2].copy()
    elif sampling == yo.S420:
        half = decode(data, "YCbCr", half=True)
        assert half.shape == (ch, cw, 3), (half.shape, ch, cw)
        cb, cr = half[..., 1].copy(), half[..., 2].copy()
        for p, c in ((cb, 1), (cr, 2)):
            assert np.array_equal(yo.upsample(sampling, p, w, h), full[..., c]), ("4:2:0 chroma", w, h)
    else:
        planes = []
        for c in (1, 2):
            rows = [solve_h2v1(full[r, :, c].astype(np.int64), cw) for r in range(h)]
            if any(r is None for r in rows):
                return None
            planes.append(np.stack(rows))
        cb, cr = planes
        for p, c in ((cb, 1), (cr, 2)):
            assert np.array_equal(yo.upsample(sampling, p, w, h), full[..., c]), ("4:2:2 chroma", w, h)
    want = np.empty((h, w, 4), np.uint8)
    want[..., 0], want[..., 1], want[..., 2], want[..., 3] = rgb[..., 2], rgb[..., 1], rgb[..., 0], 255
    return y, cb, cr, want


def main():
    arrays, names = {}, []
    for i, (w, h) in enumerate(SIZES):
        for s in yo.SAMPLINGS:
            r = case(w, h, s, seed=1000 + 7 * i + s)
            if r is None:
                print("no preimage:", w, h, yo.NAMES[s])
                continue
            name = f"{yo.NAMES[s]}_{w}x{h}"
            names.append(name)
            for k, a in zip(("y", "cb", "cr", "bgra"), r):
                arrays[f"{name}/{k}"] = a
    arrays["cases"] = np.array(names)
    arrays["libjpeg_turbo_version"] = np.array(features.version("libjpeg_turbo"))
    arrays["pillow_version"] = np.array(Image.__version__)
    arrays["weak_422"] = np.array("4:2:2 planes are a solved preimage of libjpeg-turbo's h2v1 upsampling, not decoder output")
    np.savez_compressed(OUT, **arrays)
    print(f"{len(names)} cases -> {OUT}")


if __name__ == "__main__":
    main()
