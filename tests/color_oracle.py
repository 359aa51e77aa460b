"""The reference's colour nodes, node by node, on the CPU oracle (TEST INFRASTRUCTURE).

A chain is a list of ("matrix", m[5][5]), ("enable_transparency",) and ("white_balance", threshold or None) steps.  `run_chain`
replays it the way the reference's graph does after expansion: ColorMatrixSrgb with oracle.color_matrix (color_matrix.rs:5-28),
EnableTransparency as its expand-level node (A = 255 on a Bgr32 frame, nothing on Bgra32; enable_transparency.rs:27-33), and the
white balance with oracle.white_balance (white_balance.rs:93-121).  `riapi_steps` is layout.rs:562-591 written from the reference with
the oracle's own preset matrices (oracle.color_filter_matrix); tests/test_color_oracle.py checks it against the product's
riapi_color_steps."""
import numpy as np

import oracle

SEPIA, GRAY_NTSC, GRAY_FLAT, GRAY_BT709, GRAY_RY, INVERT, ALPHA, CONTRAST, BRIGHTNESS, SATURATION = range(10)


def histograms(img: np.ndarray) -> np.ndarray:
    """histogram.rs:7-20 over every pixel: (3, 256) counters, R, G, B"""
    return np.stack([np.bincount(img[..., c].ravel(), minlength=256) for c in (2, 1, 0)]).astype(np.uint64)


def run_chain(img: np.ndarray, steps, alpha_meaningful: bool):
    """-> (the chain's result on a copy of img (h, w, 4), alpha_meaningful after it, R/G/B histograms the white balance saw or None)"""
    a = np.ascontiguousarray(img).copy()
    am, hist = bool(alpha_meaningful), None
    for s in steps:
        if s[0] == "matrix":
            oracle.color_matrix(a, s[1])
        elif s[0] == "enable_transparency":
            if not am:
                a[..., 3] = 255
                am = True
        elif s[0] == "white_balance":
            hist = histograms(a)
            oracle.white_balance(a, s[1])
        else:
            raise ValueError(s)
    return a, am, hist


def preset(which: int, p: float = 0.0):
    """the steps ColorFilterSrgb expands into (flow/nodes/color.rs:49-80)"""
    m = ("matrix", oracle.color_filter_matrix(which, p))
    return [("enable_transparency",), m] if which == ALPHA else [m]


def riapi_steps(alpha=None, brightness=None, contrast=None, saturation=None, sepia=None, grayscale=None, balance_white=None):
    out = []
    if alpha is not None:
        out += preset(ALPHA, alpha)
    if brightness is not None:
        out += preset(BRIGHTNESS, brightness)
    if contrast is not None:
        out += preset(CONTRAST, contrast)
    if saturation is not None:
        out += preset(SATURATION, saturation)
    if sepia:
        out += preset(SEPIA)
    if grayscale is not None:
        out += preset({"true": GRAY_NTSC, "ntsc": GRAY_NTSC, "y": GRAY_NTSC, "flat": GRAY_FLAT, "bt709": GRAY_BT709, "ry": GRAY_RY}[grayscale])
    if balance_white in (True, "true", "area"):
        out.append(("white_balance", None))
    return out


def of_product(steps):
    """the oracle chain of the product's step records (imageflow_b200 ColorMatrixSrgb, EnableTransparency(),
    WhiteBalanceHistogramAreaThresholdSrgb; lists flattened)"""
    out = []
    for s in steps:
        if isinstance(s, (list, tuple)):
            out += of_product(s)
        elif type(s).__name__ == "ColorMatrixSrgb":
            out.append(("matrix", np.array(s.matrix, np.float32)))
        elif type(s).__name__ == "EnableTransparency":
            out.append(("enable_transparency",))
        elif type(s).__name__ == "WhiteBalanceHistogramAreaThresholdSrgb":
            out.append(("white_balance", s.threshold))
        else:
            raise ValueError(s)
    return out
