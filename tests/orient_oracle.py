"""The reference's orientation nodes, node by node, on the CPU oracle's flips and transpose (TEST INFRASTRUCTURE).

flow/nodes/rotate_flip_transpose.rs expands ApplyOrientation { flag } into rotations, flips and transposes, and each rotation into
flips and transposes; FlipH / FlipV mutate the bitmap in place (graphics/flip.rs) and Transpose writes a new canvas of swapped size
(graphics/transpose.rs).  `run_nodes` replays such a chain with oracle.flip_horizontal / flip_vertical / transpose.  `gather` is the
closed form of include/ifb200.h, written from its table; tests/test_orient_oracle.py checks one against the other."""
import numpy as np

import oracle

ROTATE_90, ROTATE_180, ROTATE_270, FLIP_H, FLIP_V, TRANSPOSE = "Rotate90", "Rotate180", "Rotate270", "FlipH", "FlipV", "Transpose"
NODES = (ROTATE_90, ROTATE_180, ROTATE_270, FLIP_H, FLIP_V, TRANSPOSE)

# rotate_flip_transpose.rs ApplyOrientationDef::expand (any other flag: no node)
APPLY_ORIENTATION = {7: [ROTATE_180, TRANSPOSE], 8: [ROTATE_270], 6: [ROTATE_90], 5: [TRANSPOSE], 4: [FLIP_V], 3: [ROTATE_180], 2: [FLIP_H]}
# Rotate90Def / Rotate270Def / Rotate180Def::expand
ROTATION = {ROTATE_90: [FLIP_V, TRANSPOSE], ROTATE_270: [TRANSPOSE, FLIP_V], ROTATE_180: [FLIP_V, FLIP_H]}


def primitives(steps):
    """steps: node names, or ("ApplyOrientation", flag) -> the FlipH / FlipV / Transpose nodes they expand into"""
    out = []
    for s in steps:
        if isinstance(s, tuple):
            out += primitives(APPLY_ORIENTATION.get(s[1], []))
        elif s in ROTATION:
            out += primitives(ROTATION[s])
        else:
            out.append(s)
    return out


def run_nodes(img: np.ndarray, steps) -> np.ndarray:
    """the chain on a copy of img (h, w, 4) uint8, one oracle call per node"""
    a = np.ascontiguousarray(img).copy()
    for p in primitives(steps):
        if p == FLIP_H:
            oracle.flip_horizontal(a)
        elif p == FLIP_V:
            oracle.flip_vertical(a)
        else:
            t = np.zeros((a.shape[1], a.shape[0], 4), np.uint8)
            oracle.transpose(a, t)
            a = t
    return a


def gather(img: np.ndarray, o: int) -> np.ndarray:
    """out(x, y) = in(...) of the table in include/ifb200.h; flags other than 2..8 are the identity"""
    h, w = img.shape[:2]
    t = o in (5, 6, 7, 8)
    oh, ow = (w, h) if t else (h, w)
    y, x = np.indices((oh, ow))
    src = {2: (w - 1 - x, y), 3: (w - 1 - x, h - 1 - y), 4: (x, h - 1 - y), 5: (y, x), 6: (y, h - 1 - x), 7: (w - 1 - y, h - 1 - x),
           8: (w - 1 - y, x)}.get(o, (x, y))
    return img[src[1], src[0]]


def coordinate_image(w: int, h: int) -> np.ndarray:
    """(h, w, 4) uint8 whose pixel (x, y) holds x in bytes 0-1 and y in bytes 2-3 (little-endian)"""
    y, x = np.indices((h, w), dtype=np.uint32)
    return (x | (y << 16)).astype("<u4").view(np.uint8).reshape(h, w, 4)


def coordinates(img: np.ndarray):
    """the (x, y) arrays a coordinate_image's pixels carry"""
    v = np.ascontiguousarray(img).view("<u4")[..., 0]
    return v & 0xFFFF, v >> 16
