"""Python mirror of the reference's operator interface for the hot path (argument meaning and error
behaviour follow graphics/scaling.rs:19-90 and graphics/color_matrix.rs:5-28); thin marshalling over the C ABI."""
from __future__ import annotations

import ctypes as C
import enum
from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np

from ._lib import CanvasDesc, ColorDesc, ColorStep, OrientDesc, PixelConvertDesc, ResampleDesc, RoundCornersDesc, WatermarkDesc, lib


class Filter(enum.IntEnum):
    """graphics/weights.rs:45-78 (repr(C) discriminants)."""
    RobidouxFast = 1; Robidoux = 2; RobidouxSharp = 3; Ginseng = 4; GinsengSharp = 5; Lanczos = 6
    LanczosSharp = 7; Lanczos2 = 8; Lanczos2Sharp = 9; CubicFast = 10; Cubic = 11; CubicSharp = 12
    CatmullRom = 13; Mitchell = 14; CubicBSpline = 15; Hermite = 16; Jinc = 17; RawLanczos3 = 18
    RawLanczos3Sharp = 19; RawLanczos2 = 20; RawLanczos2Sharp = 21; Triangle = 22; Linear = 23; Box = 24
    CatmullRomFast = 25; CatmullRomFastSharp = 26; Fastest = 27; MitchellFast = 28; NCubic = 29
    NCubicSharp = 30; LegacyIDCTFilter = 31


class WorkingFloatspace(enum.IntEnum):
    """graphics/color.rs:4-9 (Gamma is not reachable from scale_and_render)."""
    StandardRGB = 0
    LinearRGB = 1


class BitmapCompositing(enum.IntEnum):
    """graphics/bitmaps.rs:156-160."""
    ReplaceSelf = 0
    BlendWithSelf = 1
    BlendWithMatte = 2


class ErrorKind(enum.IntEnum):
    Ok = 0; InvalidArgument = 1; MethodNotImplemented = 2; InvalidState = 3
    TotalWeightZero = 10; SourcePixelCountTooLarge = 11; NoPixelInputs = 12; BadFilter = 13; Capacity = 14
    NoDevice = 20; CudaError = 21; OutOfMemory = 22
    InvalidNodeParams = 100          # raised by the mirror's node layouts (watermark_layout), never returned by the library


class FlowError(RuntimeError):
    """Mirror of imageflow's FlowError{kind, message}."""
    def __init__(self, code: int, message: str):
        try:
            self.kind = ErrorKind(code)
        except ValueError:
            self.kind = ErrorKind.InvalidState
        self.code = code
        super().__init__(f"{self.kind.name}: {message}")


def _check(rc: int, buf) -> None:
    if rc:
        raise FlowError(rc, buf.value.decode("utf-8", "replace"))


@dataclass
class ScaleAndRenderParams:
    """graphics/scaling.rs:9-17."""
    x: int = 0
    y: int = 0
    w: int = 0
    h: int = 0
    sharpen_percent_goal: float = 0.0
    interpolation_filter: Filter = Filter.Robidoux
    scale_in_colorspace: WorkingFloatspace = WorkingFloatspace.LinearRGB


@dataclass
class BitmapWindow:
    """BitmapWindowMut<u8> for a BGRA bitmap: host (numpy) or device (raw pointer) pixels + the bits of
    BitmapInfo that scale_and_render reads (alpha_meaningful, compose; bitmaps.rs)."""
    ptr: int
    w: int
    h: int
    stride: int
    alpha_meaningful: bool = False
    compose: BitmapCompositing = BitmapCompositing.ReplaceSelf
    matte_bgra: Sequence[int] = (0, 0, 0, 0)
    pixel_layout: str = "BGRA"
    _keep: object = field(default=None, repr=False)

    @staticmethod
    def from_numpy(a: np.ndarray, **kw) -> "BitmapWindow":
        assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 4 and a.strides[2] == 1 and a.strides[1] == 4
        return BitmapWindow(a.ctypes.data, a.shape[1], a.shape[0], a.strides[0], _keep=a, **kw)

    @staticmethod
    def from_torch(t, **kw) -> "BitmapWindow":
        """t: uint8 CUDA tensor of shape (H, W, 4) (row stride may be padded)."""
        assert t.dim() == 3 and t.shape[2] == 4 and t.stride(2) == 1 and t.stride(1) == 4
        return BitmapWindow(t.data_ptr(), t.shape[1], t.shape[0], t.stride(0), _keep=t, **kw)

    def window(self, x1: int, y1: int, x2: int, y2: int) -> Optional["BitmapWindow"]:
        """bitmaps.rs:413-431: sub-rect view (None when out of bounds)."""
        if not (0 <= x1 < x2 <= self.w and 0 <= y1 < y2 <= self.h):
            return None
        return BitmapWindow(self.ptr + y1 * self.stride + x1 * 4, x2 - x1, y2 - y1, self.stride, self.alpha_meaningful,
                            self.compose, self.matte_bgra, self.pixel_layout, self._keep)


def _fill_desc(d: ResampleDesc, inp: BitmapWindow, canvas: BitmapWindow, info: ScaleAndRenderParams, color_matrix=None, keep=None) -> None:
    """Writes one job into a zero-initialised ResampleDesc (in place: descriptor arrays are filled without temporaries)."""
    if inp.pixel_layout != "BGRA" or canvas.pixel_layout != "BGRA":            # scaling.rs:43-48
        raise FlowError(ErrorKind.MethodNotImplemented, "scale_and_render only supports BGRA bitmaps")
    d.in_ = inp.ptr; d.in_w = inp.w; d.in_h = inp.h; d.in_stride = inp.stride
    d.canvas = canvas.ptr; d.cv_w = canvas.w; d.cv_h = canvas.h; d.cv_stride = canvas.stride
    d.x = info.x; d.y = info.y; d.w = info.w; d.h = info.h
    d.filter = int(info.interpolation_filter)
    d.sharpen_percent = float(info.sharpen_percent_goal)
    d.linear = 1 if info.scale_in_colorspace == WorkingFloatspace.LinearRGB else 0
    d.alpha_meaningful = 1 if inp.alpha_meaningful else 0
    d.compose = int(canvas.compose)
    m = canvas.matte_bgra
    if m[0] or m[1] or m[2] or m[3]:
        d.matte_bgra = (C.c_uint8 * 4)(*m)
    if color_matrix is not None:
        cm = np.ascontiguousarray(color_matrix, np.float32).reshape(25)
        d.color_matrix = cm.ctypes.data
        (keep if keep is not None else []).append(cm)
        d._cm = cm


def _desc(inp: BitmapWindow, canvas: BitmapWindow, info: ScaleAndRenderParams, color_matrix=None, keep=None) -> ResampleDesc:
    d = ResampleDesc()
    _fill_desc(d, inp, canvas, info, color_matrix, keep)
    return d


def scale_and_render(inp: BitmapWindow, canvas: BitmapWindow, info: ScaleAndRenderParams, color_matrix=None) -> None:
    """graphics/scaling.rs:19-90 with HOST bitmaps (the drop-in call). Raises FlowError."""
    d = _desc(inp, canvas, info, color_matrix)
    buf = C.create_string_buffer(512)
    _check(lib().ifb200_scale_and_render(C.byref(d), buf, 512), buf)


def scale_and_render_many(jobs) -> None:
    """n independent scale_and_render calls with HOST bitmaps, pipelined inside the library
    (jobs: iterable of (input, canvas, params[, color_matrix]))."""
    jobs = list(jobs)
    arr = (ResampleDesc * len(jobs))()
    keep = []
    for i, j in enumerate(jobs):
        arr[i] = _desc(j[0], j[1], j[2], j[3] if len(j) > 3 else None, keep)
    buf = C.create_string_buffer(512)
    _check(lib().ifb200_scale_and_render_many(arr, len(jobs), buf, 512), buf)


def window_bgra32_apply_color_matrix(window: BitmapWindow, m) -> None:
    """graphics/color_matrix.rs:5-28, in place on a HOST window; m is [[f32;5];5]."""
    mm = np.ascontiguousarray(m, np.float32).reshape(25)
    buf = C.create_string_buffer(512)
    _check(lib().ifb200_color_matrix_bgra8(window.ptr, window.w, window.h, window.stride,
                                            mm.ctypes.data_as(C.POINTER(C.c_float)), buf, 512), buf)


def apply_matte(window: BitmapWindow, matte_bgra) -> None:
    """graphics/blend.rs:6-59 (Bitmap::apply_matte), in place on a HOST window."""
    mm = (C.c_uint8 * 4)(*matte_bgra)
    buf = C.create_string_buffer(512)
    _check(lib().ifb200_apply_matte_bgra8(window.ptr, window.w, window.h, window.stride, mm, int(bool(window.alpha_meaningful)), buf, 512), buf)


def bitmap_window_transpose(from_window: BitmapWindow, to_window: BitmapWindow) -> None:
    """graphics/transpose.rs:95-121 on HOST windows: to[x][y] = from[y][x]; dimensions must be swapped, BGRA only."""
    if from_window.w != to_window.h or from_window.h != to_window.w or from_window.pixel_layout != to_window.pixel_layout:
        raise FlowError(ErrorKind.InvalidArgument,
                        "For transposition, canvas and input formats must be the same and dimensions must be swapped")
    if from_window.pixel_layout != "BGRA":
        raise FlowError(ErrorKind.InvalidArgument, "Only BGRA layout is supported")
    buf = C.create_string_buffer(512)
    _check(lib().ifb200_transpose_bgra8(from_window.ptr, from_window.stride, from_window.w, from_window.h,
                                        to_window.ptr, to_window.stride, buf, 512), buf)


def flow_bitmap_bgra_flip_vertical_safe(bitmap: BitmapWindow) -> None:
    """graphics/flip.rs:10-22, in place on a HOST bitmap."""
    buf = C.create_string_buffer(512)
    _check(lib().ifb200_flip_vertical_bgra8(bitmap.ptr, bitmap.w, bitmap.h, bitmap.stride, buf, 512), buf)


def flow_bitmap_bgra_flip_horizontal_safe(bitmap: BitmapWindow) -> None:
    """graphics/flip.rs:25-39, in place on a HOST bitmap."""
    buf = C.create_string_buffer(512)
    _check(lib().ifb200_flip_horizontal_bgra8(bitmap.ptr, bitmap.w, bitmap.h, bitmap.stride, buf, 512), buf)


def white_balance_srgb_mut(bitmap: BitmapWindow, threshold: Optional[float] = None) -> None:
    """flow/nodes/white_balance.rs:93-121 (WhiteBalanceHistogramAreaThresholdSrgb { threshold }), in place on a HOST bitmap."""
    buf = C.create_string_buffer(512)
    _check(lib().ifb200_white_balance_srgb_bgra8(bitmap.ptr, bitmap.w, bitmap.h, bitmap.stride, -1.0 if threshold is None else float(threshold), buf, 512), buf)


@dataclass(frozen=True)
class RoundCornersMode:
    """imageflow_types RoundCornersMode (lib.rs:1257-1268).  `kind` is the enum's declaration index (ifb200_corners_mode);
    `radius` is (top_left, top_right, bottom_right, bottom_left), the field order of the *Custom variants."""
    kind: int
    radius: tuple = (0.0, 0.0, 0.0, 0.0)
    PERCENTAGE, PIXELS, CIRCLE, PERCENTAGE_CUSTOM, PIXELS_CUSTOM = range(5)

    @classmethod
    def percentage(cls, p: float) -> "RoundCornersMode":
        return cls(cls.PERCENTAGE, (float(p), 0.0, 0.0, 0.0))

    @classmethod
    def pixels(cls, p: float) -> "RoundCornersMode":
        return cls(cls.PIXELS, (float(p), 0.0, 0.0, 0.0))

    @classmethod
    def circle(cls) -> "RoundCornersMode":
        return cls(cls.CIRCLE)

    @classmethod
    def percentage_custom(cls, top_left: float, top_right: float, bottom_right: float, bottom_left: float) -> "RoundCornersMode":
        return cls(cls.PERCENTAGE_CUSTOM, (float(top_left), float(top_right), float(bottom_right), float(bottom_left)))

    @classmethod
    def pixels_custom(cls, top_left: float, top_right: float, bottom_right: float, bottom_left: float) -> "RoundCornersMode":
        return cls(cls.PIXELS_CUSTOM, (float(top_left), float(top_right), float(bottom_right), float(bottom_left)))


def _fill_corners_desc(d: RoundCornersDesc, window: BitmapWindow, mode: RoundCornersMode, matte_bgra) -> None:
    if window.pixel_layout != "BGRA":                                          # rounded_corners.rs:192-194
        raise FlowError(ErrorKind.InvalidArgument, "Only BGRA supported for rounded corners")
    d.px = window.ptr; d.w = window.w; d.h = window.h; d.stride = window.stride
    d.mode = int(mode.kind)
    d.radius = (C.c_float * 4)(*mode.radius)
    d.matte_bgra = (C.c_uint8 * 4)(*matte_bgra)


def flow_bitmap_bgra_clear_around_rounded_corners(window: BitmapWindow, mode: RoundCornersMode, matte_bgra) -> None:
    """graphics/rounded_corners.rs:187-346, in place on a HOST window; matte_bgra = background_color as BGRA8."""
    d = RoundCornersDesc()
    _fill_corners_desc(d, window, mode, matte_bgra)
    buf = C.create_string_buffer(512)
    _check(lib().ifb200_round_corners_bgra8(C.byref(d), buf, 512), buf)


# ---------------------------------------------------------------- canvas operations (Batch.canvas), named after the imageflow_types nodes
@dataclass
class FillRect:
    """Node::FillRect { x1, y1, x2, y2, color } on `window` (bitmaps.rs:1504-1562); color = Color::to_bgra8() bytes (b, g, r, a)."""
    window: BitmapWindow
    x1: int
    y1: int
    x2: int
    y2: int
    color: Sequence[int]


@dataclass
class CopyRectToCanvas:
    """Node::CopyRectToCanvas { from_x, from_y, w, h, x, y }: copy_rectangle(input, canvas, ...) (graphics/copy_rect.rs:12-97)."""
    input: BitmapWindow
    canvas: BitmapWindow
    from_x: int
    from_y: int
    w: int
    h: int
    x: int
    y: int


@dataclass
class ExpandCanvas:
    """Node::ExpandCanvas { left, top, right, bottom, color } of `input` (clone_crop_fill_expand.rs:224-260).  The new canvas is
    allocated by Batch.canvas (a uint8 CUDA tensor, rows padded to 64 bytes as bitmaps.rs:803-804) unless `canvas` is given."""
    input: BitmapWindow
    left: int
    top: int
    right: int
    bottom: int
    color: Sequence[int]
    canvas: Optional[BitmapWindow] = None


@dataclass
class EnableTransparency:
    """EnableTransparencyMutDef (flow/nodes/enable_transparency.rs:70-86): a Bgr32 window gets A = 255 and becomes Bgra32.  With a
    window it is a canvas operation (Batch.canvas); without one, a step of a colour chain (Batch.color_chain), where it has the
    meaning of the expand-level node: nothing on a Bgra32 window (enable_transparency.rs:27-33)."""
    window: Optional[BitmapWindow] = None


def _device_of(w: BitmapWindow, default: int) -> int:
    k = w._keep
    return k.device.index if getattr(getattr(k, "device", None), "type", None) == "cuda" else default


def new_canvas(w: int, h: int, device: int = 0, alpha_meaningful: bool = True) -> BitmapWindow:
    """Bitmap::create_u8's buffer on the GPU (bitmaps.rs:803-804): an uninitialised w x h BGRA8 window of a uint8 CUDA tensor whose
    rows are padded to 64 bytes."""
    import torch
    stride = (w * 4 + 63) // 64 * 64
    t = torch.empty((h, stride // 4, 4), dtype=torch.uint8, device=torch.device("cuda", device))[:, :w]
    return BitmapWindow(t.data_ptr(), w, h, stride, alpha_meaningful, _keep=t)


def watermark_red_dot(window: BitmapWindow) -> list:
    """flow/nodes/watermark_red_dot.rs:26-39: a 3x3 FillRect of FF0000 in the bottom-right corner of frames larger than 3x3."""
    if window.w > 3 and window.h > 3:
        return [FillRect(window, window.w - 3, window.h - 3, window.w, window.h, (0, 0, 255, 255))]
    return []


def region(window: BitmapWindow, x1: int, y1: int, x2: int, y2: int, color, device: int = 0):
    """RegionDef::expand (clone_crop_fill_expand.rs:390-451): the op that makes Region { x1, y1, x2, y2, background_color } of
    `window` -- an ExpandCanvas of the cropped window, or, when the region misses the window, a FillRect of a new canvas of the
    window's format (CreateCanvas)."""
    if y2 <= y1 or x2 <= x1:
        raise FlowError(ErrorKind.InvalidArgument, f"Invalid coordinates: {x1},{y1} {x2},{y2} should describe the top-left and "
                                                   "bottom-right corners of the region in pixels. Not a rectangle.")
    if x1 >= window.w or y1 >= window.h or x2 <= 0 or y2 <= 0:
        cv = new_canvas(x2 - x1, y2 - y1, _device_of(window, device), window.alpha_meaningful)
        return FillRect(cv, 0, 0, cv.w, cv.h, tuple(color))
    crop = window.window(min(window.w, max(0, x1)), min(window.h, max(0, y1)), min(window.w, max(0, x2)), min(window.h, max(0, y2)))
    return ExpandCanvas(crop, max(0, -x1), max(0, -y1), max(0, x2 - window.w), max(0, y2 - window.h), tuple(color))


def _round_f32(v) -> int:
    """`(f32).round() as i32`: half away from zero, saturating, NaN -> 0"""
    import math
    v = float(v)
    if v != v:
        return 0
    r = math.copysign(math.floor(abs(v) + 0.5), v) if math.isfinite(v) else v
    return int(max(-2 ** 31, min(2 ** 31 - 1, r)))


def region_percent(window: BitmapWindow, left: float, top: float, right: float, bottom: float, color, device: int = 0):
    """RegionPercentDef (clone_crop_fill_expand.rs:265-350): get_coords in f32, then region()."""
    if bottom <= top or right <= left:
        raise FlowError(ErrorKind.InvalidArgument, f"Invalid coordinates: {left},{top} {right},{bottom} should describe the top-left and "
                                                   "bottom-right corners of the region in percentages. Not a rectangle.")
    f, hundred = np.float32, np.float32(100)
    x1 = _round_f32(f(window.w) * f(left) / hundred)
    y1 = _round_f32(f(window.h) * f(top) / hundred)
    x2 = _round_f32(f(window.w) * f(right) / hundred)
    y2 = _round_f32(f(window.h) * f(bottom) / hundred)
    if x2 < x1:
        x2 = x1 + 1
    if y2 < y1:
        y2 = y1 + 1
    return region(window, x1, y1, x2, y2, color, device)


_FILL_RECT, _COPY_RECT, _EXPAND, _NORMALIZE_ALPHA = range(4)          # enum ifb200_canvas_op


def _fill_canvas_desc(d: CanvasDesc, op, device: int):
    """Fills d for one op; returns the window the op writes (its metadata updated as the reference updates the bitmap's)."""
    def target(w: BitmapWindow):
        d.px = w.ptr; d.w = w.w; d.h = w.h; d.stride = w.stride; d.alpha_meaningful = int(bool(w.alpha_meaningful))

    def source(w: BitmapWindow):
        d.in_ = w.ptr; d.in_w = w.w; d.in_h = w.h; d.in_stride = w.stride; d.in_alpha_meaningful = int(bool(w.alpha_meaningful))

    wins = [getattr(op, n) for n in ("window", "input", "canvas") if getattr(op, n, None) is not None]
    if any(w.pixel_layout != "BGRA" for w in wins):
        raise FlowError(ErrorKind.InvalidArgument, "Only BGRA supported for canvas operations")
    if isinstance(op, FillRect):
        w = op.window
        if w.compose == BitmapCompositing.BlendWithMatte and (op.x1, op.y1, op.x2, op.y2) != (0, 0, w.w, w.h):   # bitmaps.rs:1512-1519
            raise FlowError(ErrorKind.InvalidArgument, "Cannot draw a rectangle on a sub-rectangle of a bitmap in BlendWithMatte mode")
        d.op = _FILL_RECT
        target(w)
        d.x1, d.y1, d.x2, d.y2 = op.x1, op.y1, op.x2, op.y2
        d.color_bgra = (C.c_uint8 * 4)(*op.color)
        return lambda: w
    if isinstance(op, CopyRectToCanvas):
        d.op = _COPY_RECT
        target(op.canvas); source(op.input)
        d.x1, d.y1, d.x2, d.y2, d.cw, d.ch = op.from_x, op.from_y, op.x, op.y, op.w, op.h

        def done(cv=op.canvas, inp=op.input):                     # copy_rect.rs:37, :47-54
            cv.compose = BitmapCompositing.BlendWithSelf
            if inp.alpha_meaningful:
                cv.alpha_meaningful = True
            return cv
        return done
    if isinstance(op, ExpandCanvas):
        d.op = _EXPAND
        inp = op.input
        w, h = inp.w + op.left + op.right, inp.h + op.top + op.bottom
        am = bool(inp.alpha_meaningful) if op.color[3] == 255 else True      # clone_crop_fill_expand.rs:239
        cv = op.canvas if op.canvas is not None else new_canvas(w, h, device)
        target(cv); source(inp)
        d.x1, d.y1, d.x2, d.y2 = op.left, op.top, op.right, op.bottom
        d.color_bgra = (C.c_uint8 * 4)(*op.color)

        def done():
            cv.alpha_meaningful = am
            cv.compose = BitmapCompositing.BlendWithSelf
            return cv
        return done
    if isinstance(op, EnableTransparency):
        w = op.window
        if w is None:
            raise FlowError(ErrorKind.InvalidArgument, "EnableTransparency as a canvas operation needs a window")
        if w.alpha_meaningful:                                   # enable_transparency.rs:74-78
            raise FlowError(ErrorKind.InvalidArgument, "Need Bgr32 input image to convert to bgra32")
        d.op = _NORMALIZE_ALPHA
        target(w)

        def done():
            w.alpha_meaningful = True
            w.compose = BitmapCompositing.BlendWithSelf
            return w
        return done
    raise FlowError(ErrorKind.InvalidArgument, f"not a canvas operation: {op!r}")


# ---------------------------------------------------------------- orientation (Batch.orient), named after the imageflow_types nodes
@dataclass(frozen=True)
class ApplyOrientation:
    """Node::ApplyOrientation { flag }: the EXIF orientation a decoder inserts after the decode (flow/nodes/codecs_and_pointer.rs)."""
    flag: int


# the unit nodes of imageflow_types
Rotate90, Rotate180, Rotate270, FlipH, FlipV, Transpose = "Rotate90", "Rotate180", "Rotate270", "FlipH", "FlipV", "Transpose"

# the reference's expansions (flow/nodes/rotate_flip_transpose.rs): ApplyOrientation by flag (any other flag: nothing), then the
# rotations into flips and transposes
_APPLY_ORIENTATION = {2: (FlipH,), 3: (Rotate180,), 4: (FlipV,), 5: (Transpose,), 6: (Rotate90,), 7: (Rotate180, Transpose), 8: (Rotate270,)}
_EXPANSION = {Rotate90: (FlipV, Transpose), Rotate180: (FlipV, FlipH), Rotate270: (Transpose, FlipV),
              FlipH: (FlipH,), FlipV: (FlipV,), Transpose: (Transpose,)}
# EXIF orientation -> (transposes, source x reversed, source y reversed): out(x, y) = in(x', y') as in include/ifb200.h
_ORIENTATION = {1: (False, False, False), 2: (False, True, False), 3: (False, True, True), 4: (False, False, True),
                5: (True, False, False), 6: (True, False, True), 7: (True, True, True), 8: (True, True, False)}


_ORIENT_DESC_DTYPE = np.dtype({"names": [n for n, _ in OrientDesc._fields_],
                               "formats": [np.uint64 if t is C.c_void_p else np.dtype(t) for n, t in OrientDesc._fields_],
                               "offsets": [getattr(OrientDesc, n).offset for n, _ in OrientDesc._fields_], "itemsize": C.sizeof(OrientDesc)})


def _primitives(steps):
    for s in steps:
        if isinstance(s, ApplyOrientation):
            yield from _primitives(_APPLY_ORIENTATION.get(int(s.flag), ()))
        elif s in _EXPANSION:
            yield from _EXPANSION[s]
        else:
            raise FlowError(ErrorKind.InvalidArgument, f"not an orientation node: {s!r}")


def _oriented(a: np.ndarray, orientation: int) -> np.ndarray:
    """the output of `orientation` on a (rows, columns) array, as a view"""
    t, fx, fy = _ORIENTATION.get(int(orientation), _ORIENTATION[1])
    b = a[::-1 if fy else 1, ::-1 if fx else 1]
    return b.swapaxes(0, 1) if t else b


def orientation_of(steps) -> int:
    """The EXIF orientation 1..8 that a chain of ApplyOrientation(flag), Rotate90, Rotate180, Rotate270, FlipH, FlipV and Transpose
    nodes amounts to: every such chain is one element of the eight symmetries of a rectangle, found here by its action on a 3 x 2
    probe."""
    probe = np.arange(6).reshape(2, 3)
    a = probe
    for p in _primitives(steps):
        a = a[:, ::-1] if p == FlipH else a[::-1] if p == FlipV else a.T
    return next(o for o in range(1, 9) if np.array_equal(_oriented(probe, o), a))


def _rust_div_rem(a: int, b: int):
    """Rust's i32 `/` (truncating) and `%` (the sign of a)"""
    q = abs(a) // abs(b) * (1 if (a >= 0) == (b >= 0) else -1)
    return q, a - b * q


def riapi_rotate_steps(degrees: int) -> list:
    """add_rotate of RIAPI's layout (imageflow_riapi ir4/layout.rs) for `rotate=` / `srotate=`: match ((rot / 90) + 4) % 4 in i32,
    so -90 is Rotate270, 45 nothing, and -450 nothing (the remainder -1 matches no arm)."""
    q, _ = _rust_div_rem(int(degrees), 90)
    _, r = _rust_div_rem(q + 4, 4)
    return [{1: Rotate90, 2: Rotate180, 3: Rotate270}[r]] if r in (1, 2, 3) else []


def riapi_flip_steps(h: bool, v: bool) -> list:
    """add_flip of RIAPI's layout for `flip=` / `sflip=` as (h, v): FlipH, then FlipV."""
    return ([FlipH] if h else []) + ([FlipV] if v else [])


def apply_orientation(window: BitmapWindow, flag: int, device: int = 0):
    """The job of Batch.orient for ApplyOrientation { flag } of `window` into a newly allocated canvas of the window's format (its
    dimensions swapped for 5..8, rows padded to 64 bytes as bitmaps.rs:803-804): (window, canvas, flag).  Batch.orient returns the
    canvas."""
    t = _ORIENTATION.get(int(flag), _ORIENTATION[1])[0]
    w, h = (window.h, window.w) if t else (window.w, window.h)
    return window, new_canvas(w, h, _device_of(window, device), window.alpha_meaningful), int(flag)


# ---------------------------------------------------------------- colour chains (Batch.color_chain), named after the imageflow_types nodes
@dataclass(eq=False)
class ColorMatrixSrgb:
    """Node::ColorMatrixSrgb { matrix }: window_bgra32_apply_color_matrix (graphics/color_matrix.rs:5-28), matrix[k][c] = the weight of
    input channel k (r, g, b, a, then the bias row) in output channel c."""
    matrix: np.ndarray

    def __post_init__(self):
        self.matrix = np.array(self.matrix, np.float32).reshape(5, 5)


@dataclass(frozen=True)
class WhiteBalanceHistogramAreaThresholdSrgb:
    """Node::WhiteBalanceHistogramAreaThresholdSrgb { threshold } (flow/nodes/white_balance.rs:93-121); None = 0.006."""
    threshold: Optional[float] = None


class ColorFilterSrgb:
    """Node::ColorFilterSrgb(filter): each preset returns the steps the node expands into (flow/nodes/color.rs:49-80) -- one
    ColorMatrixSrgb of color_filter_matrix(), preceded by EnableTransparency for Alpha."""
    @staticmethod
    def sepia(): return [ColorMatrixSrgb(color_filter_matrix(0))]
    @staticmethod
    def grayscale_ntsc(): return [ColorMatrixSrgb(color_filter_matrix(1))]
    @staticmethod
    def grayscale_flat(): return [ColorMatrixSrgb(color_filter_matrix(2))]
    @staticmethod
    def grayscale_bt709(): return [ColorMatrixSrgb(color_filter_matrix(3))]
    @staticmethod
    def grayscale_ry(): return [ColorMatrixSrgb(color_filter_matrix(4))]
    @staticmethod
    def invert(): return [ColorMatrixSrgb(color_filter_matrix(5))]
    @staticmethod
    def alpha(p: float): return [EnableTransparency(), ColorMatrixSrgb(color_filter_matrix(6, p))]
    @staticmethod
    def contrast(p: float): return [ColorMatrixSrgb(color_filter_matrix(7, p))]
    @staticmethod
    def brightness(p: float): return [ColorMatrixSrgb(color_filter_matrix(8, p))]
    @staticmethod
    def saturation(p: float): return [ColorMatrixSrgb(color_filter_matrix(9, p))]


_GRAYSCALE = {"ntsc": ColorFilterSrgb.grayscale_ntsc, "true": ColorFilterSrgb.grayscale_ntsc, "y": ColorFilterSrgb.grayscale_ntsc,
              "flat": ColorFilterSrgb.grayscale_flat, "bt709": ColorFilterSrgb.grayscale_bt709, "ry": ColorFilterSrgb.grayscale_ry}


def riapi_color_steps(alpha=None, brightness=None, contrast=None, saturation=None, sepia=None, grayscale=None, balance_white=None) -> list:
    """The colour steps RIAPI's layout emits (imageflow_riapi ir4/layout.rs:562-591) from the parsed values of s.alpha, s.brightness,
    s.contrast, s.saturation, s.sepia, s.grayscale (true / ntsc / y -> Ntsc, flat, bt709, ry) and a.balancewhite (true / area -> the
    area threshold; other algorithms emit nothing), in the reference's order."""
    steps = []
    for p, preset in ((alpha, ColorFilterSrgb.alpha), (brightness, ColorFilterSrgb.brightness), (contrast, ColorFilterSrgb.contrast),
                      (saturation, ColorFilterSrgb.saturation)):
        if p is not None:
            steps += preset(float(p))
    if sepia:
        steps += ColorFilterSrgb.sepia()
    if grayscale is not None:
        steps += _GRAYSCALE[str(grayscale).lower()]()
    if balance_white is True or str(balance_white).lower() in ("true", "area"):
        steps.append(WhiteBalanceHistogramAreaThresholdSrgb())
    return steps


_COLOR_MATRIX, _COLOR_ENABLE_TRANSPARENCY, _COLOR_WHITE_BALANCE = range(3)          # enum ifb200_color_step_kind


def _struct_dtype(S):
    def fmt(t):
        if t is C.c_void_p:
            return np.uint64
        if hasattr(t, "_length_"):
            return (np.dtype(t._type_), (t._length_,))
        return np.dtype(t)
    return np.dtype({"names": [n for n, _ in S._fields_], "formats": [fmt(t) for _, t in S._fields_],
                     "offsets": [getattr(S, n).offset for n, _ in S._fields_], "itemsize": C.sizeof(S)})


_COLOR_STEP_DTYPE, _COLOR_DESC_DTYPE = _struct_dtype(ColorStep), _struct_dtype(ColorDesc)


def _color_steps(steps):
    """-> (packed ifb200_color_step array, the array's address, whether the chain contains EnableTransparency, whether it contains a
    ColorMatrixSrgb); presets' lists are flattened"""
    flat = []
    for s in steps:
        flat.extend(s if isinstance(s, (list, tuple)) else [s])
    a = np.zeros(len(flat), _COLOR_STEP_DTYPE)
    for i, s in enumerate(flat):
        if isinstance(s, ColorMatrixSrgb):
            a[i]["kind"] = _COLOR_MATRIX; a[i]["matrix"] = s.matrix.reshape(25)
        elif isinstance(s, EnableTransparency) and s.window is None:
            a[i]["kind"] = _COLOR_ENABLE_TRANSPARENCY
        elif isinstance(s, WhiteBalanceHistogramAreaThresholdSrgb):
            a[i]["kind"] = _COLOR_WHITE_BALANCE; a[i]["threshold"] = -1.0 if s.threshold is None else float(s.threshold)
        else:
            raise FlowError(ErrorKind.InvalidArgument, f"not a colour step: {s!r}")
    return (a, a.ctypes.data, any(isinstance(s, EnableTransparency) for s in flat), any(isinstance(s, ColorMatrixSrgb) for s in flat))


# ---------------------------------------------------------------- watermarks (Batch.watermark), named after the imageflow_types records
class WatermarkConstraintMode(enum.Enum):
    """imageflow_types WatermarkConstraintMode (lib.rs:1022-1041); each maps onto the ConstraintMode of the same name."""
    Distort = "distort"; Within = "within"; Fit = "fit"; WithinCrop = "within_crop"; FitCrop = "fit_crop"


@dataclass(frozen=True)
class ConstraintGravity:
    """imageflow_types ConstraintGravity: Center (x = y = None) or Percentage { x, y } (f32 percentages)."""
    x: Optional[float] = None
    y: Optional[float] = None

    @classmethod
    def center(cls) -> "ConstraintGravity":
        return cls()

    @classmethod
    def percentage(cls, x: float, y: float) -> "ConstraintGravity":
        return cls(float(x), float(y))


@dataclass(frozen=True)
class WatermarkConstraintBox:
    """imageflow_types WatermarkConstraintBox (lib.rs:1078-1087): ImagePercentage / CanvasPercentage { x1, y1, x2, y2 } (f32) and
    ImageMargins / CanvasMargins { left, top, right, bottom } (u32), `values` in field order."""
    kind: str
    values: tuple
    IMAGE_PERCENTAGE, IMAGE_MARGINS, CANVAS_PERCENTAGE, CANVAS_MARGINS = "image_percentage", "image_margins", "canvas_percentage", "canvas_margins"

    @classmethod
    def image_percentage(cls, x1, y1, x2, y2): return cls(cls.IMAGE_PERCENTAGE, tuple(float(v) for v in (x1, y1, x2, y2)))
    @classmethod
    def canvas_percentage(cls, x1, y1, x2, y2): return cls(cls.CANVAS_PERCENTAGE, tuple(float(v) for v in (x1, y1, x2, y2)))
    @classmethod
    def image_margins(cls, left, top, right, bottom): return cls(cls.IMAGE_MARGINS, tuple(int(v) for v in (left, top, right, bottom)))
    @classmethod
    def canvas_margins(cls, left, top, right, bottom): return cls(cls.CANVAS_MARGINS, tuple(int(v) for v in (left, top, right, bottom)))


@dataclass(frozen=True)
class Watermark:
    """imageflow_types Watermark (lib.rs:1092-1101).  `hints` is accepted and, as in the reference, not used: the expansion's
    DrawImageExact gets `constraint.hints`, which is None (flow/nodes/watermark.rs:121,180)."""
    io_id: int = 0
    fit_box: Optional[WatermarkConstraintBox] = None
    fit_mode: Optional[WatermarkConstraintMode] = None
    gravity: Optional[ConstraintGravity] = None
    min_canvas_width: Optional[int] = None
    min_canvas_height: Optional[int] = None
    opacity: Optional[float] = None
    hints: object = None


@dataclass(frozen=True)
class WatermarkDraw:
    """What WatermarkDef::expand emits for one frame: Crop { crop } of the watermark (None: no crop), ColorFilterSrgb::Alpha(opacity)
    (None: no opacity step) and DrawImageExact { x, y, w, h } with the filter scale_render.rs:251-259 picks for hints None; no sharpen,
    linear light."""
    crop: Optional[tuple]
    x: int
    y: int
    w: int
    h: int
    filter: Filter
    opacity: Optional[float]


_F32 = np.float32
_I32_MAX = 2 ** 31 - 1


def _round_f64(v: float) -> float:
    """f64::round: half away from zero (exact: x - trunc(x) has no rounding error)"""
    import math
    if not math.isfinite(v):
        return v
    t = float(math.trunc(v))
    if abs(v - t) >= 0.5:
        t += math.copysign(1.0, v)
    return t


def _clamp_f32(v, lo: float, hi: float):
    """f32::clamp: NaN stays NaN"""
    v = _F32(v)
    return v if v != v else _F32(min(max(v, _F32(lo)), _F32(hi)))


class _LayoutError(Exception):
    pass


class _Ratio:
    """sizing.rs AspectRatio: a size and the ratio it stands for"""
    __slots__ = ("w", "h")

    def __init__(self, w: int, h: int):
        if w < 1 or h < 1:
            raise _LayoutError(f"InvalidDimensions {w}x{h}")
        self.w, self.h = int(w), int(h)

    def ratio(self) -> float:
        return float(self.w) / float(self.h)

    def aspect_wider_than(self, o: "_Ratio") -> bool:
        return o.ratio() > self.ratio()

    def loss_w(self, tw: int) -> float:
        rounded_y = _round_f64(float(self.h) * (float(tw) / float(self.w)))
        return abs(float(tw) - rounded_y * self.ratio())

    def loss_h(self, th: int) -> float:
        rounded_x = _round_f64(float(self.w) * (float(th) / float(self.h)))
        return abs(float(th) - rounded_x / self.ratio())

    def proportional(self, basis: int, basis_is_width: bool, target: Optional["_Ratio"]) -> int:
        """sizing.rs:118-184, f64 throughout"""
        import sys
        snap = 1.0 - sys.float_info.epsilon
        if target is not None:
            snap = self.loss_h(target.h) if basis_is_width else self.loss_w(target.w)
        ratio = self.ratio()
        snap_a = self.h if basis_is_width else self.w
        snap_b = (target.h if basis_is_width else target.w) if target is not None else snap_a
        fl = float(basis) / ratio if basis_is_width else ratio * float(basis)
        da, db = fl - float(snap_a), fl - float(snap_b)
        if abs(da) <= snap and abs(da) <= abs(db):
            v = snap_a
        elif abs(db) <= snap:
            v = snap_b
        else:
            r = _round_f64(fl)
            if r <= -2.0 ** 31 or r >= float(_I32_MAX):
                raise _LayoutError("ValueScalingFailed")
            v = int(r)
        if v < 0:
            raise _LayoutError("ValueScalingFailed")
        return 1 if v == 0 else v

    def box_of(self, target: "_Ratio", inner: bool) -> "_Ratio":
        if target.aspect_wider_than(self) == inner:
            return _Ratio(target.w, self.proportional(target.w, True, target))
        return _Ratio(self.proportional(target.h, False, target), target.h)

    def intersection(self, o: "_Ratio") -> "_Ratio":
        return _Ratio(min(self.w, o.w), min(self.h, o.h))

    def distort_with(self, old: "_Ratio", new: "_Ratio") -> "_Ratio":
        def mult(v, num, den):                                 # i64 multiply and truncating divide, then `as i32`
            q = abs(v * num) // abs(den) * (1 if (v * num >= 0) == (den > 0) else -1)
            return (q + 2 ** 31) % 2 ** 32 - 2 ** 31
        return _Ratio(mult(self.w, new.w, old.w), mult(self.h, new.h, old.h))


def _cmp(a: int, b: int) -> int:
    return (a > b) - (a < b)


# The sizing steps of the five watermark modes (Ir4Layout::get_instructions + build_constraints, layout.rs:162-332): (FitMode, ScaleMode)
# = Distort (Stretch, Both), Within (Max, DownscaleOnly), Fit (Max, Both), WithinCrop (Crop, DownscaleOnly), FitCrop (Crop, Both).
# Conditions compare the canvas with the target (sizing.rs:433-435): ("either", 1) = Cond::Either(Greater), ("either", -1) = Either(Less),
# ("l1s1",) = Larger1DSmaller1D.
_MODE_STEPS = {
    WatermarkConstraintMode.Distort: [("distort",)],
    WatermarkConstraintMode.Within: [("skip_unless", ("either", 1)), ("scale_inner",)],
    WatermarkConstraintMode.Fit: [("scale_inner",)],
    WatermarkConstraintMode.WithinCrop: [("skip_if", ("either", -1)), ("scale_outer",), ("crop",), ("begin",), ("skip_unless", ("l1s1",)),
                                         ("crop_intersection",)],
    WatermarkConstraintMode.FitCrop: [("scale_outer",), ("crop",)],
}


def _ir4_gravity1d(p, inner: int, outer: int) -> int:
    """Ir4Layout::gravity1d (layout.rs:673-683): f32, clamped to [0, outer - inner]"""
    if (outer < inner and inner < 1) or outer < 1:
        raise _LayoutError("align")
    ratio = _clamp_f32(p, 0.0, 100.0) / _F32(100)
    return max(0, min(_round_f32(_F32(outer - inner) * ratio), outer - inner))


def _gravity_xy(gravity: Optional[ConstraintGravity]):
    return (50.0, 50.0) if gravity is None or gravity.x is None else (gravity.x, gravity.y)


def process_constraint(src_w: int, src_h: int, mode: WatermarkConstraintMode, w: int, h: int, gravity: Optional[ConstraintGravity] = None):
    """Ir4Layout::process_constraint (imageflow_riapi ir4/layout.rs:334-412) for the modes a watermark can ask for, with both w and h
    given: -> (crop [x1, y1, x2, y2] of the source or None, scale_to (w, h)).  The reference panics (unwrap) on a layout error; here it
    is FlowError(InvalidState)."""
    try:
        initial = _Ratio(src_w, src_h)
        target = _Ratio(w, h)                                  # get_ideal_target_size with w, h >= 1 and zoom 1 (layout.rs:93-131)
        lay = {"source": initial, "target": target, "canvas": initial, "image": initial}

        def crop_to(t: _Ratio):
            if t.w > lay["canvas"].w or t.h > lay["canvas"].h:
                raise _LayoutError("ImpossibleCrop")
            img = lay["image"].intersection(t)
            lay.update(source=img.box_of(lay["source"], True), image=img, canvas=t)

        def cond(c) -> bool:
            cw, ch = _cmp(lay["canvas"].w, target.w), _cmp(lay["canvas"].h, target.h)
            return (cw == c[1] or ch == c[1]) if c[0] == "either" else (cw, ch) in ((1, -1), (-1, 1))

        skipping = False
        for st in _MODE_STEPS[WatermarkConstraintMode(mode)]:
            if st[0] == "skip_if" and cond(st[1]) or st[0] == "skip_unless" and not cond(st[1]):
                skipping = True
            elif st[0] == "begin":
                skipping = False
            if skipping or st[0] in ("skip_if", "skip_unless", "begin"):
                continue
            if st[0] in ("scale_inner", "scale_outer"):
                cv = lay["canvas"].box_of(target, st[0] == "scale_inner")
                lay.update(image=lay["image"].distort_with(lay["canvas"], cv), canvas=cv)
            elif st[0] == "distort":
                lay.update(image=lay["image"].distort_with(lay["canvas"], target), canvas=target)
            elif st[0] == "crop":
                crop_to(target)
            else:                                              # crop_intersection
                crop_to(lay["image"].intersection(target))
        new_crop = lay["source"]
        gx, gy = _gravity_xy(gravity)
        cx, cy = _ir4_gravity1d(gx, new_crop.w, initial.w), _ir4_gravity1d(gy, new_crop.h, initial.h)
    except _LayoutError as e:
        raise FlowError(ErrorKind.InvalidState, f"watermark layout failed: {e}") from None
    crop = None
    if cx > 0 or cy > 0 or (new_crop.w, new_crop.h) != (initial.w, initial.h):
        crop = [cx, cy, cx + new_crop.w, cy + new_crop.h]
    return crop, (lay["image"].w, lay["image"].h)


def _i32(v: int) -> int:
    return (int(v) + 2 ** 31) % 2 ** 32 - 2 ** 31


def _fit_box(w: int, h: int, fit_box: Optional[WatermarkConstraintBox]):
    """WatermarkDef::get_bounding_box (watermark.rs:11-58): (x1, y1, x2, y2), or None when the box is not at least 1x1"""
    if fit_box is None:
        return 0, 0, w, h
    if fit_box.kind in (WatermarkConstraintBox.IMAGE_MARGINS, WatermarkConstraintBox.CANVAS_MARGINS):
        left, top, right, bottom = fit_box.values
        if (left + right) % 2 ** 32 < w and (top + bottom) % 2 ** 32 < h:          # u32 addition
            return _i32(left), _i32(top), w - _i32(right), h - _i32(bottom)
        return None

    def px(p, c):
        return _round_f32((_clamp_f32(p, 0.0, 100.0) / _F32(100)) * _F32(c))
    x1, y1, x2, y2 = fit_box.values
    x1, y1, x2, y2 = px(x1, w), px(y1, h), px(x2, w), px(y2, h)
    return (x1, y1, x2, y2) if x1 < x2 and y1 < y2 else None


def _wm_gravity1d(p, inner: int, outer: int) -> int:
    """WatermarkDef::gravity1d (watermark.rs:59-66): f32, NOT clamped (unlike Ir4Layout's)"""
    if (outer < inner and inner < 1) or outer < 1:
        raise FlowError(ErrorKind.InvalidNodeParams, "Watermark fit_box does not work")
    return _round_f32(_F32(outer - inner) * (_clamp_f32(p, 0.0, 100.0) / _F32(100)))


def watermark_layout(frame_w: int, frame_h: int, wm_w: int, wm_h: int, watermark: Watermark) -> Optional[WatermarkDraw]:
    """WatermarkDef::expand (flow/nodes/watermark.rs:96-205) for a frame_w x frame_h frame and a wm_w x wm_h watermark: None when the
    node deletes itself (the frame is not strictly larger than min_canvas_*, or the fit box is under 1x1), else the draw.  Raises
    FlowError(InvalidNodeParams) where WatermarkDef::gravity1d fails."""
    if not (_i32(watermark.min_canvas_width or 0) < frame_w and _i32(watermark.min_canvas_height or 0) < frame_h):
        return None
    box = _fit_box(frame_w, frame_h, watermark.fit_box)
    if box is None:
        return None
    bx1, by1, bx2, by2 = box
    mode = watermark.fit_mode if watermark.fit_mode is not None else WatermarkConstraintMode.Within
    crop, (w, h) = process_constraint(wm_w, wm_h, mode, (bx2 - bx1) % 2 ** 32, (by2 - by1) % 2 ** 32, watermark.gravity)
    gx, gy = _gravity_xy(watermark.gravity)
    x = _wm_gravity1d(gx, w, bx2 - bx1) + bx1
    y = _wm_gravity1d(gy, h, by2 - by1) + by1
    op = 1.0 if watermark.opacity is None else _clamp_f32(watermark.opacity, 0.0, 1.0)
    in_w, in_h = (crop[2] - crop[0], crop[3] - crop[1]) if crop is not None else (wm_w, wm_h)
    filt = Filter.Ginseng if (w > in_w or h > in_h) else Filter.Robidoux          # scale_render.rs:251-259, hints None
    return WatermarkDraw(tuple(crop) if crop is not None else None, x, y, w, h, filt, float(op) if op < 1 else None)


def riapi_watermark_placement(watermarks) -> tuple:
    """RIAPI's layout (imageflow_riapi ir4/layout.rs:593-636): the watermarks drawn before the padding (fit box None, ImageMargins,
    ImagePercentage) and after it (CanvasMargins, CanvasPercentage), each in the given order."""
    wms = list(watermarks or [])
    before = [w for w in wms if w.fit_box is None or w.fit_box.kind in (WatermarkConstraintBox.IMAGE_MARGINS, WatermarkConstraintBox.IMAGE_PERCENTAGE)]
    after = [w for w in wms if w.fit_box is not None and w.fit_box.kind in (WatermarkConstraintBox.CANVAS_MARGINS, WatermarkConstraintBox.CANVAS_PERCENTAGE)]
    return before, after


_WATERMARK_DESC_DTYPE = np.dtype({
    "names": ["draw_" + n for n, _ in ResampleDesc._fields_] + ["opacity"],
    "formats": [np.uint64 if t is C.c_void_p else (np.uint8, (4,)) if hasattr(t, "_length_") else np.dtype(t) for _, t in ResampleDesc._fields_]
               + [np.float32],
    "offsets": [WatermarkDesc.draw.offset + getattr(ResampleDesc, n).offset for n, _ in ResampleDesc._fields_] + [WatermarkDesc.opacity.offset],
    "itemsize": C.sizeof(WatermarkDesc)})


def flow_scale_spatial(samples: np.ndarray, n: int, srgb: bool = False) -> np.ndarray:
    """flow_scale_spatial[_srgb]_{n}x{n} (c_components/lib/codecs_jpeg_idct_fast.c) applied to every 8x8 block of a plane of
    samples (H x W uint8, both multiples of 8; host memory): returns the (H/8*n) x (W/8*n) plane."""
    a = np.ascontiguousarray(samples, np.uint8)
    h, w = a.shape
    if h % 8 or w % 8:
        raise FlowError(int(ErrorKind.InvalidArgument), "plane dimensions must be multiples of 8")
    out = np.zeros((h // 8 * n, w // 8 * n) if 1 <= n <= 7 else (1, 1), np.uint8)
    buf = C.create_string_buffer(512)
    _check(lib().ifb200_block_scale_u8(a.ctypes.data, a.strides[0], w // 8, h // 8, out.ctypes.data, out.strides[0], n, int(bool(srgb)), buf, 512), buf)
    return out


def detect_content(bitmap: BitmapWindow, threshold: int = 1):
    """graphics/whitespace.rs:284-331 with a HOST bitmap -> (x1, y1, x2, y2)."""
    rect = (C.c_uint32 * 4)()
    buf = C.create_string_buffer(512)
    _check(lib().ifb200_detect_content_bgra8(bitmap.ptr, bitmap.w, bitmap.h, bitmap.stride, int(bool(bitmap.alpha_meaningful)), int(threshold), rect, buf, 512), buf)
    return tuple(rect)


def detect_content_from_codes(codes: np.ndarray):
    """host half of detect_content alone: the reference's window walk over a (h, w) uint8 code map (ifb_whitespace.h);
    no CUDA call.  -> ((x1, y1, x2, y2), pixels visited)"""
    codes = np.ascontiguousarray(codes, np.uint8)
    rect = (C.c_uint32 * 4)(); n = C.c_uint64()
    rc = lib().ifb200_detect_content_from_codes(codes.ctypes.data, codes.shape[1], codes.shape[0], rect, C.byref(n))
    if rc:
        raise FlowError(rc, "empty or oversized code map")
    return tuple(rect), n.value


def color_filter_matrix(which: int, p: float = 0.0) -> np.ndarray:
    """flow/nodes/color.rs:86-225 presets (0 sepia ... 9 saturation)."""
    m = np.zeros(25, np.float32)
    rc = lib().ifb200_color_filter_matrix(which, p, m.ctypes.data_as(C.POINTER(C.c_float)))
    if rc:
        raise FlowError(rc, "unknown colour filter")
    return m.reshape(5, 5)


def populate_weights(filter: int, out_size: int, in_size: int, kernel_width_scale: float = 1.0,
                     lobe_mode: int = 0, lobe_value: float = 0.0):
    """graphics/weights.rs:681-788 -> [(left_pixel, right_pixel, weights f32[])] per output pixel."""
    left = np.zeros(out_size, np.uint32); right = np.zeros(out_size, np.uint32); off = np.zeros(out_size + 1, np.uint32)
    cap = out_size * (int(2 * (6.5 * max(1.0, in_size / max(out_size, 1)) * max(kernel_width_scale, 1.0))) + 8)
    w = np.zeros(cap, np.float32)
    u32p, f32p = C.POINTER(C.c_uint32), C.POINTER(C.c_float)
    rc = lib().ifb200_weights(int(filter), kernel_width_scale, lobe_mode, lobe_value, out_size, in_size,
                              left.ctypes.data_as(u32p), right.ctypes.data_as(u32p), off.ctypes.data_as(u32p),
                              w.ctypes.data_as(f32p), cap)
    if rc:
        raise FlowError(rc, "populate_weights failed")
    return [(int(left[i]), int(right[i]), w[off[i]:off[i + 1]].copy()) for i in range(out_size)]


def plan_probe(geometries, threads: int = 1, want_hash: bool = False) -> dict:
    """Host-side cost of preparing kernel tables: builds (and discards) the plans of `geometries` =
    [(in_w, in_h, out_w, out_h[, filter[, sharpen_percent]])] on `threads` host threads.  No CUDA call."""
    arr = (ResampleDesc * len(geometries))()
    for d, g in zip(arr, geometries):
        d.in_w, d.in_h, d.w, d.h = g[:4]
        d.filter = g[4] if len(g) > 4 else int(Filter.Robidoux)
        d.sharpen_percent = g[5] if len(g) > 5 else 0.0
    sec, nb, hs = C.c_double(), C.c_uint64(), C.c_uint64()
    buf = C.create_string_buffer(512)
    _check(lib().ifb200_plan_probe(arr, len(geometries), threads, C.byref(sec), C.byref(nb), C.byref(hs) if want_hash else None, buf, 512), buf)
    return {"seconds": sec.value, "table_bytes": nb.value, "table_hash": hs.value if want_hash else None}


# ---------------------------------------------------------------- pixel formats at the graph's edges (Batch.pixel_convert)
@dataclass
class PixelRows:
    """Rows of 1, 2, 3 or 4 interleaved uint8 channels (Gray8, GrayAlpha8, RGB24, RGBA32 or BGRA32) at any row stride and any byte
    offset: what a decoder hands over and an encoder takes.  Host (numpy) or device (raw pointer) memory, like BitmapWindow."""
    ptr: int
    w: int
    h: int
    stride: int
    channels: int
    _keep: object = field(default=None, repr=False)

    @staticmethod
    def _of(ptr, shape, strides, keep) -> "PixelRows":
        if len(shape) != 3 or shape[2] not in (1, 2, 3, 4) or strides[2] != 1 or strides[1] != shape[2] or strides[0] < 0:
            raise FlowError(ErrorKind.InvalidArgument, f"pixel rows must be (H, W, C) uint8 with C in 1..4, interleaved, rows of any "
                                                       f"non-negative stride; got shape {tuple(shape)}, strides {tuple(strides)}")
        return PixelRows(ptr, shape[1], shape[0], strides[0], shape[2], keep)

    @staticmethod
    def from_numpy(a: np.ndarray) -> "PixelRows":
        if a.dtype != np.uint8:
            raise FlowError(ErrorKind.InvalidArgument, f"pixel rows must be uint8, not {a.dtype}")
        return PixelRows._of(a.ctypes.data, a.shape, a.strides, a)

    @staticmethod
    def from_torch(t) -> "PixelRows":
        """t: uint8 CUDA tensor of shape (H, W, C), e.g. nvJPEG's interleaved RGB; a CHW tensor needs .permute(1, 2, 0).contiguous()."""
        import torch
        if t.dtype != torch.uint8:
            raise FlowError(ErrorKind.InvalidArgument, f"pixel rows must be uint8, not {t.dtype}")
        return PixelRows._of(t.data_ptr(), tuple(t.shape), t.stride(), t)

    @staticmethod
    def of(x) -> "PixelRows":
        """PixelRows of a numpy array, a torch tensor, a BitmapWindow (4 channels) or PixelRows"""
        if isinstance(x, PixelRows):
            return x
        if isinstance(x, BitmapWindow):
            return PixelRows(x.ptr, x.w, x.h, x.stride, 4, x._keep)
        return PixelRows.from_numpy(x) if isinstance(x, np.ndarray) else PixelRows.from_torch(x)


# op -> (source channels, destination channels), include/ifb200.h enum ifb200_pixel_op
_PIXEL_OP_CHANNELS = {0: (3, 4), 1: (4, 4), 2: (1, 4), 3: (2, 4), 4: (4, 3)}


@dataclass
class RgbToBgra:
    """rgb_to_bgra (graphics/swizzle.rs:26-31): RGB24 rows -> BGRA, alpha 255 (image_png_decoder.rs, jpeg_decoder.rs)."""
    src: object
    dst: object
    opaque: bool = False
    OP = 0


@dataclass
class RgbaToBgra:
    """copy_swap_br (graphics/swizzle.rs:14-19): bytes 0 and 2 swapped, so RGBA -> BGRA and BGRA -> RGBA alike.  dst None = in place
    (swap_br_inplace, :8-12); opaque = alpha 255 (the encoders' swap then fill, zen_encoder.rs:585-603, in one pass)."""
    src: object
    dst: object = None
    opaque: bool = False
    OP = 1


@dataclass
class GrayToBgra:
    """gray_to_bgra (graphics/swizzle.rs:33-37): Gray8 rows -> (v, v, v, 255)."""
    src: object
    dst: object
    opaque: bool = False
    OP = 2


@dataclass
class GrayAlphaToBgra:
    """gray_alpha_to_bgra (graphics/swizzle.rs:39-45): GrayAlpha8 rows -> (v, v, v, a); opaque = alpha 255."""
    src: object
    dst: object
    opaque: bool = False
    OP = 3


@dataclass
class BgraToRgb:
    """to_vec_rgb (graphics/bitmaps.rs:1316-1345): BGRA -> RGB24 rows, alpha dropped without a matte."""
    src: object
    dst: object
    opaque: bool = False
    OP = 4


_PIXEL_OPS = {c.OP: c for c in (RgbToBgra, RgbaToBgra, GrayToBgra, GrayAlphaToBgra, BgraToRgb)}
_PIXEL_DESC_DTYPE = np.dtype({"names": [n for n, _ in PixelConvertDesc._fields_],
                              "formats": [np.uint64 if t is C.c_void_p else np.dtype(t) for n, t in PixelConvertDesc._fields_],
                              "offsets": [getattr(PixelConvertDesc, n).offset for n, _ in PixelConvertDesc._fields_],
                              "itemsize": C.sizeof(PixelConvertDesc)})


def pixel_op_for(channels: int, to_bgra: bool = True):
    """The record that converts rows of `channels` channels into BGRA (to_bgra) or BGRA into them (3: BgraToRgb, 4: RgbaToBgra)."""
    ops = {1: GrayToBgra, 2: GrayAlphaToBgra, 3: RgbToBgra, 4: RgbaToBgra} if to_bgra else {3: BgraToRgb, 4: RgbaToBgra}
    if channels not in ops:
        raise FlowError(ErrorKind.InvalidArgument, f"no conversion {'from' if to_bgra else 'to'} {channels}-channel rows")
    return ops[channels]


def device_count() -> int:
    return lib().ifb200_device_count()


class Batch:
    """Device-resident batch executor (ifb200_batch_*): many independent scale_and_render calls whose
    bitmaps already live in HBM of one GPU, enqueued on a CUDA stream."""
    OPT_FORCE_GENERIC, OPT_STRIP_COLUMNS, OPT_MIN_ITEMS = 1, 2, 3

    def __init__(self, device: int = 0):
        self._h = C.c_void_p()
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_create(device, C.byref(self._h), buf, 512), buf)
        self.device = device
        self._keep = []

    def ring_status(self):
        """(usable, reason): whether the streaming ring kernel (the fast path of down-scales) can run on this device"""
        buf = C.create_string_buffer(256)
        ok = lib().ifb200_batch_ring_status(self._h, buf, 256)
        return bool(ok), buf.value.decode()

    def set_option(self, option: int, value: int) -> None:
        rc = lib().ifb200_batch_set_option(self._h, option, value)
        if rc:
            raise FlowError(rc, f"bad option {option}={value}")

    def make_descs(self, jobs):
        """jobs: iterable of (input BitmapWindow, canvas BitmapWindow, ScaleAndRenderParams[, color_matrix])."""
        jobs = list(jobs)
        arr = (ResampleDesc * len(jobs))()
        keep = []
        for i, j in enumerate(jobs):
            _fill_desc(arr[i], j[0], j[1], j[2], j[3] if len(j) > 3 else None, keep)
        keep.append([(j[0]._keep, j[1]._keep) for j in jobs])          # the bitmaps stay alive until sync() / close()
        return arr, keep

    STREAM_OWN = C.c_void_p(-1)

    @classmethod
    def _stream(cls, stream):
        """An int is a cudaStream_t (0 = the legacy default stream); "own" = the batch's private non-blocking stream
        (IFB200_STREAM_OWN, the one sync() waits for).  None = the stream the caller's tensors live on: torch's current stream
        when torch is loaded with CUDA -- work enqueued there is ordered after whatever produced the inputs and before whatever
        reads the outputs -- otherwise the batch's own stream."""
        if stream == "own":
            return cls.STREAM_OWN
        if stream is None:
            import sys
            torch = sys.modules.get("torch")
            if torch is not None and torch.cuda.is_available() and torch.cuda.is_initialized():
                return C.c_void_p(torch.cuda.current_stream().cuda_stream)
            return cls.STREAM_OWN
        return C.c_void_p(stream)

    def enqueue(self, descs, stream=None, keep=None) -> None:
        if keep:
            self._keep.append(keep)
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_enqueue(self._h, descs, len(descs), self._stream(stream), buf, 512), buf)

    def scale_and_render_many(self, jobs, stream=None) -> None:
        descs, keep = self.make_descs(jobs)
        self.enqueue(descs, stream, keep)

    def color_matrix(self, dev_ptr: int, w: int, h: int, stride: int, m, stream=None) -> None:
        mm = np.ascontiguousarray(m, np.float32).reshape(25)
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_color_matrix(self._h, dev_ptr, w, h, stride, mm.ctypes.data_as(C.POINTER(C.c_float)),
                                                self._stream(stream), buf, 512), buf)

    def transpose(self, from_window: BitmapWindow, to_window: BitmapWindow, stream=None) -> None:
        """graphics/transpose.rs:95-121 on DEVICE windows (asynchronous on `stream`)."""
        if from_window.w != to_window.h or from_window.h != to_window.w:
            raise FlowError(ErrorKind.InvalidArgument,
                            "For transposition, canvas and input formats must be the same and dimensions must be swapped")
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_transpose(self._h, from_window.ptr, from_window.stride, from_window.w, from_window.h,
                                            to_window.ptr, to_window.stride, self._stream(stream), buf, 512), buf)

    def block_scale(self, dev_in: int, in_stride: int, blocks_x: int, blocks_y: int, dev_out: int, out_stride: int, n: int, srgb: bool, stream=None) -> None:
        """flow_scale_spatial[_srgb]_{n}x{n} over a device-resident plane of 8x8 sample blocks"""
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_block_scale(self._h, dev_in, in_stride, blocks_x, blocks_y, dev_out, out_stride, n, int(bool(srgb)), self._stream(stream), buf, 512), buf)

    def white_balance(self, bitmap: BitmapWindow, threshold: Optional[float] = None, stream=None) -> None:
        """flow/nodes/white_balance.rs:93-121 on a DEVICE bitmap, in place (three kernels, asynchronous on `stream`)."""
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_white_balance(self._h, bitmap.ptr, bitmap.w, bitmap.h, bitmap.stride,
                                                -1.0 if threshold is None else float(threshold), self._stream(stream), buf, 512), buf)

    def detect_content(self, bitmap: BitmapWindow, threshold: int = 1, stream=None):
        """graphics/whitespace.rs:284-331 on a DEVICE bitmap -> (x1, y1, x2, y2); synchronises `stream`."""
        rect = (C.c_uint32 * 4)()
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_detect_content(self._h, bitmap.ptr, bitmap.w, bitmap.h, bitmap.stride, int(bool(bitmap.alpha_meaningful)),
                                                 int(threshold), rect, self._stream(stream), buf, 512), buf)
        return tuple(rect)

    def whitespace_codes(self, bitmap: BitmapWindow, dev_codes_ptr: int, threshold: int = 1, stream=None) -> None:
        """the GPU half of detect_content alone (graphics/whitespace.rs:426-613 per pixel): code map of a DEVICE bitmap into a
        DEVICE buffer of w*h bytes; asynchronous on `stream`."""
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_whitespace_codes(self._h, bitmap.ptr, bitmap.w, bitmap.h, bitmap.stride, int(bool(bitmap.alpha_meaningful)),
                                                   int(threshold), dev_codes_ptr, self._stream(stream), buf, 512), buf)

    def round_corners(self, jobs, stream=None) -> None:
        """graphics/rounded_corners.rs:187-346 on DEVICE windows, in place, all jobs in one kernel launch (asynchronous on
        `stream`).  jobs: iterable of (BitmapWindow, RoundCornersMode, matte_bgra); no two windows may share a pixel."""
        jobs = list(jobs)
        arr = (RoundCornersDesc * len(jobs))()
        for d, (window, mode, matte) in zip(arr, jobs):
            _fill_corners_desc(d, window, mode, matte)
        self._keep.append([j[0]._keep for j in jobs])
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_round_corners(self._h, arr, len(jobs), self._stream(stream), buf, 512), buf)

    def canvas(self, ops, stream=None) -> list:
        """Canvas operations on DEVICE windows, all in one kernel launch (none when no op writes a pixel), asynchronous on `stream`.
        ops: FillRect, CopyRectToCanvas, ExpandCanvas, EnableTransparency.  No op may write what another op of the call reads or
        writes.  Returns, per op, the window it wrote (ExpandCanvas: the new canvas), with alpha_meaningful and compose updated as
        the reference updates the bitmap; nothing is changed when an argument is rejected."""
        ops = list(ops)
        arr = (CanvasDesc * len(ops))()
        done = [_fill_canvas_desc(d, op, self.device) for d, op in zip(arr, ops)]
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_canvas(self._h, arr, len(ops), self._stream(stream), buf, 512), buf)
        out = [f() for f in done]
        self._keep.append([[getattr(op, n, None) for n in ("window", "input", "canvas")] for op in ops] + [w._keep for w in out])
        return out

    def orient(self, jobs, stream=None) -> list:
        """EXIF orientations on DEVICE windows, one read and one write per pixel, all jobs in one kernel launch (none when no job
        writes a pixel), asynchronous on `stream`.  jobs: iterable of (input, output or None for in place, orientation); compose a
        chain of nodes into one orientation with orientation_of().  The output is w x h for 1..4 and h x w for 5..8; in place needs
        1..4.  No job may write what another job of the call reads or writes.  Returns the output windows (with the input's
        alpha_meaningful); nothing is changed when an argument is rejected."""
        jobs = list(jobs)
        outs = []
        for inp, out, o in jobs:
            out = inp if out is None else out
            t = _ORIENTATION.get(int(o), _ORIENTATION[1])[0]
            if (out.w, out.h) != ((inp.h, inp.w) if t else (inp.w, inp.h)) or inp.pixel_layout != "BGRA" or out.pixel_layout != "BGRA":
                raise FlowError(ErrorKind.InvalidArgument, f"orientation {o} of a {inp.w}x{inp.h} BGRA window needs a "
                                                           f"{'%dx%d' % ((inp.h, inp.w) if t else (inp.w, inp.h))} BGRA output, not {out.w}x{out.h}")
            outs.append(out)
        a = np.zeros(len(jobs), _ORIENT_DESC_DTYPE)               # filled a column at a time: no per-field ctypes marshalling
        a["in_"] = [j[0].ptr for j in jobs]; a["in_w"] = [j[0].w for j in jobs]; a["in_h"] = [j[0].h for j in jobs]
        a["in_stride"] = [j[0].stride for j in jobs]; a["out"] = [o.ptr for o in outs]; a["out_stride"] = [o.stride for o in outs]
        a["orientation"] = [int(j[2]) for j in jobs]
        arr = (OrientDesc * len(jobs)).from_buffer(a)
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_orient(self._h, arr, len(jobs), self._stream(stream), buf, 512), buf)
        for (inp, _, _), out in zip(jobs, outs):
            out.alpha_meaningful = inp.alpha_meaningful
        self._keep.append([(j[0]._keep, o._keep) for j, o in zip(jobs, outs)])
        return outs

    def pixel_convert(self, jobs, stream=None) -> list:
        """Pixel-format conversions on DEVICE rows, all jobs in one kernel launch (none when no job has pixels), asynchronous on
        `stream`.  jobs: iterable of RgbToBgra, RgbaToBgra, GrayToBgra, GrayAlphaToBgra and BgraToRgb records, whose src and dst are
        BitmapWindows (BGRA) or anything PixelRows.of() takes, with the channels the op reads and writes.  No job may write what
        another job of the call reads or writes.  Returns the destinations (the source for an in-place RgbaToBgra); a BitmapWindow
        destination gets alpha_meaningful as a decoder sets it (RGBA and GrayAlpha sources, unless opaque).  Nothing is changed when
        an argument is rejected."""
        jobs = list(jobs)
        srcs, dsts = [], []
        for j in jobs:
            if not isinstance(j, tuple(_PIXEL_OPS.values())):
                raise FlowError(ErrorKind.InvalidArgument, f"not a pixel conversion: {j!r}")
            dst = j.src if j.dst is None else j.dst
            s, d = PixelRows.of(j.src), PixelRows.of(dst)
            cs, cd = _PIXEL_OP_CHANNELS[j.OP]
            if (s.channels, d.channels) != (cs, cd) or (s.w, s.h) != (d.w, d.h):
                raise FlowError(ErrorKind.InvalidArgument, f"{type(j).__name__} converts {cs}-channel rows into {cd}-channel rows of the "
                                                           f"same size, not {s.w}x{s.h}x{s.channels} into {d.w}x{d.h}x{d.channels}")
            srcs.append(s); dsts.append(d)
        a = np.zeros(len(jobs), _PIXEL_DESC_DTYPE)                # filled a column at a time: no per-field ctypes marshalling
        a["op"] = [j.OP for j in jobs]; a["opaque"] = [int(bool(j.opaque)) for j in jobs]
        a["src"] = [s.ptr for s in srcs]; a["src_stride"] = [s.stride for s in srcs]
        a["dst"] = [d.ptr for d in dsts]; a["dst_stride"] = [d.stride for d in dsts]
        a["w"] = [s.w for s in srcs]; a["h"] = [s.h for s in srcs]
        arr = (PixelConvertDesc * len(jobs)).from_buffer(a)
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_pixel_convert(self._h, arr, len(jobs), self._stream(stream), buf, 512), buf)
        out = []
        for j in jobs:
            dst = j.src if j.dst is None else j.dst
            if isinstance(dst, BitmapWindow) and j.OP != BgraToRgb.OP:
                dst.alpha_meaningful = j.OP in (RgbaToBgra.OP, GrayAlphaToBgra.OP) and not j.opaque
            out.append(dst)
        self._keep.append([(s._keep, d._keep) for s, d in zip(srcs, dsts)])
        return out

    def to_bgra(self, rows, opaque: bool = False, stream=None) -> "BitmapWindow":
        """One call from decoder rows -- an (H, W, C) uint8 CUDA tensor, C in 1..4, or PixelRows -- to a new BGRA BitmapWindow on the
        batch's device (a torch tensor with rows padded to 64 bytes, as bitmaps.rs:803-804)."""
        import torch
        s = PixelRows.of(rows)
        op = pixel_op_for(s.channels)
        pitch = (s.w * 4 + 63) // 64 * 64
        t = torch.empty((s.h, pitch // 4, 4), dtype=torch.uint8, device=f"cuda:{self.device}")[:, :s.w]
        win = BitmapWindow.from_torch(t)
        self.pixel_convert([op(s, win, opaque)], stream)
        return win

    def from_bgra(self, window: "BitmapWindow", channels: int = 3, opaque: bool = False, stream=None):
        """One call from a BGRA window to a new contiguous (H, W, channels) uint8 CUDA tensor: RGB24 (3) or RGBA32 (4) rows, as an
        encoder takes them."""
        import torch
        t = torch.empty((window.h, window.w, channels), dtype=torch.uint8, device=f"cuda:{self.device}")
        self.pixel_convert([pixel_op_for(channels, to_bgra=False)(window, t, opaque)], stream)
        return t

    def color_chain(self, jobs, stream=None) -> list:
        """Colour chains on DEVICE windows, in place, all jobs in one kernel launch (three when a job white-balances; none when no
        job writes a pixel), asynchronous on `stream`.  jobs: iterable of (window, steps), steps a list of ColorMatrixSrgb,
        EnableTransparency(), WhiteBalanceHistogramAreaThresholdSrgb and ColorFilterSrgb presets (see riapi_color_steps), applied in
        order.  No two windows may share a pixel.  Returns the windows with the metadata the nodes leave behind: BlendWithSelf
        compositing after any ColorMatrixSrgb (ColorMatrixSrgbMutDef, flow/nodes/color.rs:29) and on a Bgr32 window that met
        EnableTransparency, which is Bgra32 from then on (enable_transparency.rs:80-82); zero-area windows too, as the nodes still run
        there.  White balance leaves the metadata alone.  Nothing is changed when an argument is rejected."""
        jobs = list(jobs)
        packed = {}
        for _, steps in jobs:                                     # a steps list shared by many jobs is packed once
            if id(steps) not in packed:
                packed[id(steps)] = _color_steps(steps)
        wins = [j[0] for j in jobs]
        if any(w.pixel_layout != "BGRA" for w in wins):
            raise FlowError(ErrorKind.InvalidArgument, "Only BGRA supported for colour chains")
        a = np.zeros(len(jobs), _COLOR_DESC_DTYPE)               # filled a column at a time: no per-field ctypes marshalling
        a["px"] = [w.ptr for w in wins]; a["w"] = [w.w for w in wins]; a["h"] = [w.h for w in wins]
        a["stride"] = [w.stride for w in wins]; a["alpha_meaningful"] = [bool(w.alpha_meaningful) for w in wins]
        chains = [packed[id(j[1])] for j in jobs]
        a["steps"] = [c[1] for c in chains]; a["n_steps"] = [len(c[0]) for c in chains]
        arr = (ColorDesc * len(jobs)).from_buffer(a)
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_color_chain(self._h, arr, len(jobs), self._stream(stream), buf, 512), buf)
        for w, (_, _, et, matrix) in zip(wins, chains):
            if et and not w.alpha_meaningful:
                w.alpha_meaningful = True
                w.compose = BitmapCompositing.BlendWithSelf
            if matrix:
                w.compose = BitmapCompositing.BlendWithSelf
        self._keep.append([w._keep for w in wins])
        return wins

    def watermark(self, jobs, stream=None) -> list:
        """Watermark nodes on DEVICE frames (flow/nodes/watermark.rs), byte for byte as the reference's expansion, asynchronous on
        `stream`.  jobs: iterable of (frame, watermark window, Watermark); the watermark window is the decoded watermark (its
        alpha_meaningful is its format) and is never written.  Each job runs watermark_layout; a job whose node deletes itself changes
        nothing.  Jobs of one frame run in order as successive library calls (one per watermark a frame has), each call one resample per
        distinct watermark image and one composite launch for all its frames.  Returns the frames, drawn ones BlendWithSelf from then on
        (scale_render.rs:314).  Every layout is checked before the first call: a job the layout rejects changes nothing."""
        jobs = list(jobs)
        self.watermark_enqueue(self.make_watermark_descs(jobs), stream)
        return [j[0] for j in jobs]

    def make_watermark_descs(self, jobs) -> list:
        """The library calls of watermark(jobs), prepared: [(ifb200_watermark_desc array, frames, kept objects)], one per watermark a
        frame has.  watermark_enqueue() submits them (the frames' compose and matte are read then).  Every distinct (watermark, frame
        size, Watermark) is laid out once, and the descriptor columns are filled from per-layout arrays, so the cost per frame is a few
        dictionary lookups."""
        ents, index, eidx, frames = [], {}, [], []             # one entry per distinct (watermark, frame size, spec): (src, layout) or None
        lw = ls = None; lfw = lfh = le = -1
        for frame, wm, spec in jobs:
            if frame.pixel_layout != "BGRA":
                raise FlowError(ErrorKind.InvalidArgument, "Only BGRA supported for watermarks")
            if not (wm is lw and spec is ls and frame.w == lfw and frame.h == lfh):      # a run of one watermark costs no lookup
                k = (id(wm), frame.w, frame.h, id(spec))
                le = index.get(k)
                if le is None:
                    le = index[k] = len(ents)
                    ents.append(self._watermark_entry(frame, wm, spec))
                lw, ls, lfw, lfh = wm, spec, frame.w, frame.h
            eidx.append(le)
            frames.append(frame)
        live = [i for i, e in enumerate(eidx) if ents[e] is not None] if any(e is None for e in ents) else range(len(jobs))
        ptrs = [frames[i].ptr for i in live]
        if len(set(ptrs)) == len(ptrs):                        # every frame once: one call
            calls = [list(live)]
        else:                                                  # the k-th watermark of a frame goes into call k
            calls, seen = [], {}
            for i, p in zip(live, ptrs):
                c = seen.get(p, 0)
                seen[p] = c + 1
                if c == len(calls):
                    calls.append([])
                calls[c].append(i)
        m = max(len(ents), 1)
        col = {k: np.zeros(m, t) for k, t in (("in_", np.uint64), ("in_w", np.uint32), ("in_h", np.uint32), ("in_stride", np.uint32),
                                             ("am", np.int32), ("cv_w", np.uint32), ("cv_h", np.uint32), ("x", np.uint32),
                                             ("y", np.uint32), ("w", np.uint32), ("h", np.uint32), ("filter", np.int32), ("opacity", np.float32))}
        for e, ent in enumerate(ents):
            if ent is None:
                continue
            (src, lay), fw, fh = ent
            for k, v in (("in_", src.ptr), ("in_w", src.w), ("in_h", src.h), ("in_stride", src.stride), ("am", bool(src.alpha_meaningful)),
                         ("cv_w", fw), ("cv_h", fh), ("x", lay.x), ("y", lay.y), ("w", lay.w), ("h", lay.h), ("filter", int(lay.filter)),
                         ("opacity", 1.0 if lay.opacity is None else lay.opacity)):
                col[k][e] = v
        e_all = np.asarray(eidx, np.int64)
        out = []
        for sel in calls:
            E = e_all[np.asarray(sel, np.int64)]
            fr = [frames[i] for i in sel]
            a = np.zeros(len(sel), _WATERMARK_DESC_DTYPE)      # filled a column at a time: no per-field ctypes marshalling
            for k in ("in_", "in_w", "in_h", "in_stride", "cv_w", "cv_h", "x", "y", "w", "h", "filter"):
                a["draw_" + k] = col[k][E]
            a["draw_alpha_meaningful"] = col["am"][E]; a["opacity"] = col["opacity"][E]
            a["draw_canvas"] = [f.ptr for f in fr]; a["draw_cv_stride"] = [f.stride for f in fr]; a["draw_linear"] = 1
            out.append((a, fr, [ents[e][0][0]._keep for e in set(E.tolist())]))
        return out

    @staticmethod
    def _watermark_entry(frame: BitmapWindow, wm: BitmapWindow, spec: "Watermark"):
        """((cropped watermark window, WatermarkDraw), frame w, frame h), or None when the node deletes itself"""
        if wm.pixel_layout != "BGRA":
            raise FlowError(ErrorKind.InvalidArgument, "Only BGRA supported for watermarks")
        lay = watermark_layout(frame.w, frame.h, wm.w, wm.h, spec)
        if lay is None:
            return None
        if lay.x < 0 or lay.y < 0 or lay.x + lay.w > frame.w or lay.y + lay.h > frame.h:      # scale_render.rs:236-238
            raise FlowError(ErrorKind.InvalidNodeParams, f"DrawImageExact target rect x1={lay.x},y1={lay.y},w={lay.w},h={lay.h} "
                                                         f"does not fit canvas size {frame.w}x{frame.h}.")
        src = wm.window(*lay.crop) if lay.crop is not None else wm
        if src is None:
            raise FlowError(ErrorKind.InvalidArgument, f"crop {lay.crop} is outside the {wm.w}x{wm.h} watermark")
        return (src, lay), frame.w, frame.h

    def watermark_enqueue(self, calls, stream=None) -> None:
        """Submits make_watermark_descs(): each call takes the frames' compose and matte as they are when it is made (a frame is
        BlendWithSelf after its first watermark)."""
        self_mode = BitmapCompositing.BlendWithSelf
        for a, fr, keep in calls:
            comp = [f.compose for f in fr]
            if all(c is self_mode for c in comp):
                a["draw_compose"] = 1
            else:
                a["draw_compose"] = [int(c) for c in comp]
                for i, c in enumerate(comp):
                    if c == BitmapCompositing.BlendWithMatte:
                        a["draw_matte_bgra"][i] = tuple(fr[i].matte_bgra)
            arr = (WatermarkDesc * len(fr)).from_buffer(a)
            buf = C.create_string_buffer(512)
            _check(lib().ifb200_batch_watermark(self._h, arr, len(fr), self._stream(stream), buf, 512), buf)
            for f in fr:
                f.compose = self_mode
            self._keep.append(([f._keep for f in fr], keep))

    def flip_vertical(self, bitmap: BitmapWindow, stream=None) -> None:
        """graphics/flip.rs:10-22 on a DEVICE bitmap, in place."""
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_flip_vertical(self._h, bitmap.ptr, bitmap.w, bitmap.h, bitmap.stride, self._stream(stream), buf, 512), buf)

    def flip_horizontal(self, bitmap: BitmapWindow, stream=None) -> None:
        """graphics/flip.rs:25-39 on a DEVICE bitmap, in place."""
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_flip_horizontal(self._h, bitmap.ptr, bitmap.w, bitmap.h, bitmap.stride, self._stream(stream), buf, 512), buf)

    def sync(self) -> None:
        buf = C.create_string_buffer(512)
        _check(lib().ifb200_batch_sync(self._h, buf, 512), buf)
        import sys
        torch = sys.modules.get("torch")
        if torch is not None and torch.cuda.is_available() and torch.cuda.is_initialized():
            torch.cuda.synchronize(self.device)          # work enqueued on torch's streams (the default for stream=None)
        self._keep.clear()

    def host_profile(self) -> dict:
        """seconds the calling thread has spent inside enqueue calls so far, by part (ifb200_batch_host_profile)"""
        v = (C.c_double * 8)()
        lib().ifb200_batch_host_profile(self._h, v, 8)
        return {"enqueue_s": v[0], "plans_s": v[1], "staging_slots_s": v[2], "staging_memcpy_s": v[3], "table_uploads_s": v[4],
                "table_uploads": int(v[5]), "staged_bytes": int(v[6]), "pinned_allocs": int(v[7])}

    @property
    def kernel_launches(self) -> int:
        return lib().ifb200_batch_kernel_launches(self._h)

    @property
    def fused_jobs(self) -> int:
        return lib().ifb200_batch_fused_jobs(self._h)

    @property
    def generic_jobs(self) -> int:
        return lib().ifb200_batch_generic_jobs(self._h)

    @property
    def tile_jobs(self) -> int:
        return lib().ifb200_batch_tile_jobs(self._h)

    def close(self) -> None:
        if self._h:
            lib().ifb200_batch_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
