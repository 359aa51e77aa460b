"""python tests/golden/make_ycbcr_enc_golden.py: writes tests/golden/ycbcr_enc_golden.npz, libjpeg-turbo's compressor colour stage
(RGB -> YCbCr and chroma downsampling, as it runs on JCS_EXT_BGRA input) pinned against Pillow's bundled libjpeg-turbo.  Needs Pillow
and the CPU oracle (oracle/, for the matte cases); the tests read only the .npz.

Pillow cannot return the compressor's planes, but a JPEG stream is a deterministic function of them, so each case is checked through
streams, all at quality 100 (every quantiser 1, so that planes differing anywhere give different streams):
  Aligned sizes (both sides multiples of 16, the largest MCU):
    stream A  Pillow encodes the RGB image at the sampling;
    stream B  Pillow encodes a "YCbCr" image (libjpeg's null colour conversion) at the same sampling: Y is tests/ycbcr_enc_oracle.py's
              Y, Cb and Cr its downsampled chroma replicated back to full resolution -- libjpeg's box average of a replicated box is
              the sample itself at either bias.
    A == B byte for byte pins the oracle's colour conversion and downsampling in the interior.
  Ragged sizes: A and B differ at the padding blocks (libjpeg downsamples them from replicated full-resolution columns; the
    replicated-chroma image pads differently), so the edge rule is pinned instead: the ragged image, and the same image padded by edge
    replication to a multiple of 16, are encoded and both decoded as "YCbCr" at DCT scale 1/2, which leaves 4:2:0 chroma at its stored
    resolution (the trick of make_ycbcr_golden.py; 4:2:2 and 4:4:4 chroma come out scaled).  Their visible chroma must agree, and the padded image must pass the aligned check; the case is then the oracle on the padded image, cropped.
    The half-scale decodes disagree on some ragged cases for two reasons, neither of them in the visible samples the oracle pins:
      - 4:2:0: below the last row pair, libjpeg pads the chroma at its downsampled resolution by repeating the last downsampled row
        (jcprepct.c, expand_bottom_edge after downsampling), while the padded image's extra rows are full-resolution replicas whose
        boxes differ from that row.  The last chroma block's padding, hence its DCT, differs, and visible samples decode 1 apart.
      - 4:2:2: at DCT scale 1/2 libjpeg-turbo cannot keep the chroma unscaled in one direction only, so it decodes it at 4 x 4 and
        upsamples it horizontally with h2v1 fancy upsampling, whose neighbour past the ragged image's last chroma column is that
        column itself, while the padded image has a real one.  The columns next to the edge decode differently.
    Such cases are reported and not written; the file lists them ("dropped").
Matte cases ("m" suffix): a cut-out alpha (0, 255 and partial values) flattened by the CPU oracle of apply_matte over a non-white
matte; the stored source keeps its alpha, and the checks above run on the flattened image."""
import io
import os
import sys

import numpy as np
from PIL import Image, ImageFile, features

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from tests import ycbcr_enc_oracle as eo  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ycbcr_enc_golden.npz")
RAGGED = [(1, 1), (2, 2), (1, 9), (13, 1), (2, 7), (3, 3), (4, 5), (5, 3), (6, 2), (7, 11), (8, 8), (9, 16), (16, 9), (17, 17),
          (31, 6), (37, 23), (64, 48), (101, 7), (7, 101), (128, 96), (250, 33)]
ALIGNED = [(16, 16), (32, 48), (64, 16), (128, 96), (240, 32)]
MATTE_SIZES = [(16, 16), (37, 23), (64, 48)]
MATTE = (40, 200, 90, 255)
PIL_SUBSAMPLING = {eo.S444: 0, eo.S422: 1, eo.S420: 2}
QUALITY = 100


def image(w, h, seed, alpha=False):
    """a seeded BGRA image with smooth colour and noise; with `alpha` a cut-out: 0 and 255 regions and partial values between"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    base = np.stack([128 + 120 * np.sin(xx / 5.0 + c + seed) * np.cos(yy / 7.0 - c) for c in range(3)], axis=-1)
    out = np.empty((h, w, 4), np.uint8)
    out[..., :3] = np.clip(base + rng.normal(0, 40, (h, w, 3)), 0, 255).astype(np.uint8)
    out[..., 3] = 255
    if alpha:
        a = rng.integers(0, 256, (h, w))
        a[(xx + yy) % 5 == 0] = 0
        a[(xx * 3 + yy) % 7 == 0] = 255
        out[..., 3] = a
    return out


def encode(arr, mode, sampling):
    buf = io.BytesIO()
    Image.fromarray(arr, mode).save(buf, "JPEG", quality=QUALITY, subsampling=PIL_SUBSAMPLING[sampling])
    return buf.getvalue()


def rgb_of(bgra):
    return np.ascontiguousarray(bgra[..., 2::-1])


def replicated(sampling, y, cb, cr):
    """the "YCbCr" image whose libjpeg downsampling gives back cb and cr"""
    h, w = y.shape
    fy, fx = (2 if sampling == eo.S420 else 1), (1 if sampling == eo.S444 else 2)
    up = [np.repeat(np.repeat(c, fy, 0), fx, 1)[:h, :w] for c in (cb, cr)]
    return np.stack([y, up[0], up[1]], axis=-1)


def half_decode(data):
    """the YCbCr decode at DCT scale 1/2 (Image.draft, forced for every size)"""
    im = Image.open(io.BytesIO(data))
    d, e, o, a = im.tile[0]
    im._mode = "YCbCr"
    im.tile = [ImageFile._Tile(d, (e[0], e[1], (e[2] + 1) // 2, (e[3] + 1) // 2), o, ("YCbCr", ""))]
    im._size = ((im.size[0] + 1) // 2, (im.size[1] + 1) // 2)
    im.decoderconfig = (2, 0)
    return np.asarray(im)


def aligned_ok(sampling, flat):
    y, cb, cr = eo.convert(sampling, flat)
    return encode(rgb_of(flat), "RGB", sampling) == encode(replicated(sampling, y, cb, cr), "YCbCr", sampling)


def case(w, h, sampling, seed, matte):
    """(source, y, cb, cr) or None when the checks do not pin the case"""
    src = image(w, h, seed, alpha=matte)
    flat = eo.flatten(src, MATTE, True) if matte else src
    pw, ph = -(-w // 16) * 16, -(-h // 16) * 16
    padded = np.pad(flat, ((0, ph - h), (0, pw - w), (0, 0)), mode="edge")
    if not aligned_ok(sampling, padded):
        return None
    if (pw, ph) != (w, h):
        a, b = half_decode(encode(rgb_of(flat), "RGB", sampling)), half_decode(encode(rgb_of(padded), "RGB", sampling))
        hh, hw = a.shape[:2]
        if not np.array_equal(a[..., 1:], b[:hh, :hw, 1:]):
            return None
    y, cb, cr = eo.convert(sampling, padded)
    ch, cw = eo.chroma_shape(sampling, w, h)
    return src, y[:h, :w].copy(), cb[:ch, :cw].copy(), cr[:ch, :cw].copy()


def main():
    arrays, names, dropped = {}, [], []
    sizes = [(w, h, False) for w, h in ALIGNED + RAGGED] + [(w, h, True) for w, h in MATTE_SIZES]
    for i, (w, h, m) in enumerate(sizes):
        for s in eo.SAMPLINGS:
            name = f"{eo.NAMES[s]}_{w}x{h}" + ("m" if m else "")
            if name in names:
                continue
            r = case(w, h, s, seed=2000 + 7 * i + s, matte=m)
            if r is None:
                dropped.append(name)
                print("not pinned:", name)
                continue
            names.append(name)
            for k, a in zip(("bgra", "y", "cb", "cr"), r):
                arrays[f"{name}/{k}"] = a
    arrays["cases"] = np.array(names)
    arrays["dropped"] = np.array(dropped, dtype=str)
    arrays["matte_bgra"] = np.array(MATTE, np.uint8)
    arrays["libjpeg_turbo_version"] = np.array(features.version("libjpeg_turbo"))
    arrays["pillow_version"] = np.array(Image.__version__)
    arrays["quality"] = np.array(QUALITY)
    np.savez_compressed(OUT, **arrays)
    print(f"{len(names)} cases -> {OUT}; not pinned: {dropped}")


if __name__ == "__main__":
    main()
