"""numpy oracle of the canvas operations (TEST INFRASTRUCTURE ONLY): a plain transcription of the reference's
    BitmapWindowMut::fill_rectangle        graphics/bitmaps.rs:1504-1562
    BitmapWindowMut::normalize_unused_alpha graphics/bitmaps.rs:1564-1576
    copy_rectangle                          graphics/copy_rect.rs:12-97 (32-bit formats)
    Bitmap::create_u8's canvas fill         graphics/bitmaps.rs:829-837 (CreateCanvas)
and of the graph rewrites built on them: ExpandCanvasDef::expand (flow/nodes/clone_crop_fill_expand.rs:224-260), RegionDef /
RegionPercentDef (:265-451) and WatermarkRedDot (flow/nodes/watermark_red_dot.rs:26-39).

A window is a view of a flat byte buffer (Win), so that tests can place windows inside larger bitmaps full of sentinel bytes.
A window may carry a `mask` (one bool per 4-byte word of its buffer), in which the functions mark every pixel the reference writes."""
from __future__ import annotations

import math

import numpy as np


class CanvasArgError(ValueError):
    """ErrorKind::InvalidArgument of the reference (or, for a zero-size copy, its panic)."""


class Win:
    """A BGRA8 window of the flat uint8 buffer `buf`: w x h pixels from byte `off`, rows `stride` bytes apart."""

    def __init__(self, buf: np.ndarray, off: int, w: int, h: int, stride: int, alpha_meaningful: bool = False, mask=None):
        assert buf.ndim == 1 and buf.dtype == np.uint8 and off % 4 == 0 and stride % 4 == 0
        self.buf, self.off, self.w, self.h, self.stride, self.alpha_meaningful = buf, off, w, h, stride, alpha_meaningful
        self.mask = mask

    @staticmethod
    def of(a: np.ndarray, alpha_meaningful: bool = False) -> "Win":
        """the whole of a C-contiguous (h, w, 4) array"""
        assert a.flags.c_contiguous and a.ndim == 3 and a.shape[2] == 4
        return Win(a.reshape(-1), 0, a.shape[1], a.shape[0], a.shape[1] * 4, alpha_meaningful)

    def px(self) -> np.ndarray:
        """(h, w, 4) view of the pixels"""
        return np.lib.stride_tricks.as_strided(self.buf[self.off:], (self.h, self.w, 4), (self.stride, 4, 1))

    def sub(self, x1, y1, x2, y2) -> "Win":
        """bitmaps.rs:413-431 window(): None when empty or out of bounds"""
        if not (x1 < x2 <= self.w and y1 < y2 <= self.h):
            return None
        return Win(self.buf, self.off + y1 * self.stride + x1 * 4, x2 - x1, y2 - y1, self.stride, self.alpha_meaningful, self.mask)

    def mark(self, x1=0, y1=0, x2=None, y2=None, mask=None):
        mask = self.mask if mask is None else mask
        if mask is None:
            return
        x2 = self.w if x2 is None else x2
        y2 = self.h if y2 is None else y2
        for y in range(y1, y2):
            s = (self.off + y * self.stride) // 4
            mask[s + x1:s + x2] = True


def hex_bgra(s: str):
    """ColorSrgb::Hex ("RRGGBB" or "RRGGBBAA") as Color::to_bgra8() bytes (b, g, r, a)"""
    s = s.lstrip("#")
    r, g, b = (int(s[i:i + 2], 16) for i in (0, 2, 4))
    a = int(s[6:8], 16) if len(s) == 8 else 255
    return (b, g, r, a)


TRANSPARENT = (0, 0, 0, 0)                       # Color::Transparent


def fill_rectangle(win: Win, color, x, y, x2, y2):
    if y2 == y or x2 == x:                       # :1520-1522
        return
    if y2 <= y or x2 <= x or x2 > win.w or y2 > win.h:
        raise CanvasArgError(f"Coordinates {x},{y} {x2},{y2} must be within image dimensions {win.w}x{win.h}")
    win.px()[y:y2, x:x2] = np.array(color, np.uint8)
    win.mark(x, y, x2, y2)


def normalize_unused_alpha(win: Win):
    if win.alpha_meaningful:
        return
    win.px()[:, :, 3] = 255                      # set_alpha_to_255, row by row
    win.mark()


def copy_rectangle(inp: Win, canvas: Win, from_x, from_y, to_x, to_y, w, h):
    """copy_rect.rs:12-97; canvas.alpha_meaningful is updated as :51 updates the canvas bitmap"""
    if inp.w <= from_x or inp.h <= from_y or inp.w < from_x + w or inp.h < from_y + h or canvas.w < to_x + w or canvas.h < to_y + h:
        raise CanvasArgError("Invalid argument to copy_rect")
    if not canvas.alpha_meaningful and inp.alpha_meaningful:      # Bgr32 canvas, Bgra32 input (:47-54)
        normalize_unused_alpha(canvas)
        canvas.alpha_meaningful = True
    if not inp.alpha_meaningful and canvas.alpha_meaningful:          # Bgr32 input, Bgra32 canvas (:64-66)
        normalize_unused_alpha(inp)
    src = inp.sub(from_x, from_y, from_x + w, from_y + h)
    dst = canvas.sub(to_x, to_y, to_x + w, to_y + h)
    if src is None or dst is None:               # .window(..).unwrap() panics on an empty window (:68-79)
        raise CanvasArgError("zero-size copy")
    dst.px()[...] = src.px()                     # raw bytes, row by row (:82-97)
    dst.mark()


def create_canvas(canvas: Win, color):
    """Bitmap::create_u8 with BlendWithMatte(color) (bitmaps.rs:829-837) into an existing buffer: the buffer is zeroed
    (aligned_buffer.rs:16-42) and filled with the colour unless it is Color::Transparent"""
    canvas.px()[...] = 0
    canvas.mark()
    if tuple(color) != TRANSPARENT:
        fill_rectangle(canvas, color, 0, 0, canvas.w, canvas.h)


def expand_canvas(inp: Win, canvas: Win, left, top, right, bottom, color):
    """ExpandCanvasDef::expand: CreateCanvas(w + left + right, h + top + bottom, format, color) then CopyRectToCanvas(0, 0, left,
    top, w, h).  canvas: the buffer of the new canvas (its alpha_meaningful is set here by :239's format rule)."""
    assert canvas.w == inp.w + left + right and canvas.h == inp.h + top + bottom
    canvas.alpha_meaningful = inp.alpha_meaningful if color[3] == 255 else True
    create_canvas(canvas, color)
    copy_rectangle(inp, canvas, 0, 0, left, top, inp.w, inp.h)


def watermark_red_dot(w, h):
    """the FillRect (x1, y1, x2, y2, bgra) that WatermarkRedDot becomes on a w x h frame, or None"""
    if w > 3 and h > 3:
        return (w - 3, h - 3, w, h, hex_bgra("FF0000"))
    return None


def region(w, h, x1, y1, x2, y2):
    """RegionDef::expand on a w x h input: ("canvas", cw, ch) for a bare CreateCanvas of the input's format, or
    ("expand", (cx1, cy1, cx2, cy2), (left, top, right, bottom)) for Crop + ExpandCanvas"""
    if y2 <= y1 or x2 <= x1:
        raise CanvasArgError("not a rectangle")
    if x1 >= w or y1 >= h or x2 <= 0 or y2 <= 0:
        return ("canvas", x2 - x1, y2 - y1)
    crop = (min(w, max(0, x1)), min(h, max(0, y1)), min(w, max(0, x2)), min(h, max(0, y2)))
    return ("expand", crop, (max(0, -x1), max(0, -y1), max(0, x2 - w), max(0, y2 - h)))


def _f32_round_i32(v: np.float32) -> int:
    """`v.round() as i32` for an f32: halves away from zero, saturating"""
    v = float(v)
    if math.isnan(v):
        return 0
    r = math.floor(abs(v) + 0.5) if math.isfinite(v) else abs(v)
    r = -r if v < 0 else r
    return int(min(max(r, -2 ** 31), 2 ** 31 - 1))


def region_percent_coords(w, h, left, top, right, bottom):
    """RegionPercentDef::get_coords"""
    f = np.float32
    x1 = _f32_round_i32(f(w) * f(left) / f(100))
    y1 = _f32_round_i32(f(h) * f(top) / f(100))
    x2 = _f32_round_i32(f(w) * f(right) / f(100))
    y2 = _f32_round_i32(f(h) * f(bottom) / f(100))
    if x2 < x1:
        x2 = x1 + 1
    if y2 < y1:
        y2 = y1 + 1
    return x1, y1, x2, y2


def run_region(img: np.ndarray, alpha_meaningful: bool, x1, y1, x2, y2, color):
    """Region on a whole (h, w, 4) image: -> (new image, alpha_meaningful)"""
    h, w = img.shape[:2]
    kind, *rest = region(w, h, x1, y1, x2, y2)
    if kind == "canvas":
        out = np.empty((rest[1], rest[0], 4), np.uint8)
        create_canvas(Win.of(out), color)
        return out, alpha_meaningful
    (cx1, cy1, cx2, cy2), (l, t, r, b) = rest
    src = Win.of(np.ascontiguousarray(img), alpha_meaningful).sub(cx1, cy1, cx2, cy2)
    out = np.empty((src.h + t + b, src.w + l + r, 4), np.uint8)
    cv = Win.of(out)
    expand_canvas(src, cv, l, t, r, b, color)
    return out, cv.alpha_meaningful
