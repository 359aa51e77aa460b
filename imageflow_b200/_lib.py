"""ctypes binding of libifb200.so (include/ifb200.h).  Fails loudly when the library is missing:
there is no Python/CPU fallback for any compute entry point."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("IFB200_LIB") or os.path.join(_HERE, "libifb200.so")   # IFB200_LIB: A/B builds during development

# every symbol include/ifb200.h declares (tests/test_boundary.py checks the header against this list)
SYMBOLS = [
    "ifb200_abi_version", "ifb200_status_name", "ifb200_device_count", "ifb200_weights",
    "ifb200_byte_to_float_table", "ifb200_linear_to_srgb_table", "ifb200_color_filter_matrix", "ifb200_plan_probe",
    "ifb200_scale_and_render", "ifb200_scale_and_render_many", "ifb200_color_matrix_bgra8", "ifb200_apply_matte_bgra8", "ifb200_batch_apply_matte",
    "ifb200_transpose_bgra8", "ifb200_flip_vertical_bgra8", "ifb200_flip_horizontal_bgra8",
    "ifb200_batch_transpose", "ifb200_batch_flip_vertical", "ifb200_batch_flip_horizontal",
    "ifb200_white_balance_srgb_bgra8", "ifb200_batch_white_balance",
    "ifb200_detect_content_bgra8", "ifb200_batch_detect_content", "ifb200_detect_content_from_codes", "ifb200_batch_whitespace_codes", "ifb200_set_dropin_device",
    "ifb200_batch_create", "ifb200_batch_enqueue", "ifb200_batch_color_matrix", "ifb200_batch_sync",
    "ifb200_batch_destroy", "ifb200_batch_set_option", "ifb200_batch_kernel_launches", "ifb200_batch_host_profile",
    "ifb200_batch_fused_jobs", "ifb200_batch_generic_jobs", "ifb200_batch_tile_jobs", "ifb200_batch_ring_status", "ifb200_hv_plan_tables",
    "ifb200_block_scale_u8", "ifb200_batch_block_scale", "ifb200_round_corners_bgra8", "ifb200_batch_round_corners",
    "ifb200_batch_canvas", "ifb200_batch_orient", "ifb200_batch_color_chain", "ifb200_batch_watermark",
    "ifb200_batch_pixel_convert", "ifb200_batch_enqueue_oriented", "ifb200_batch_enqueue_rows", "ifb200_batch_detect_content_many",
    "ifb200_batch_enqueue_rows_oriented", "ifb200_batch_transform_to_srgb", "ifb200_source_profile_plan",
    "ifb200_batch_enqueue_profiled", "ifb200_batch_ycbcr_to_bgra", "ifb200_batch_bgra_to_ycbcr",
]


class ResampleDesc(C.Structure):
    """struct ifb200_resample_desc"""
    _fields_ = [
        ("in_", C.c_void_p), ("in_w", C.c_uint32), ("in_h", C.c_uint32), ("in_stride", C.c_uint32),
        ("canvas", C.c_void_p), ("cv_w", C.c_uint32), ("cv_h", C.c_uint32), ("cv_stride", C.c_uint32),
        ("x", C.c_uint32), ("y", C.c_uint32), ("w", C.c_uint32), ("h", C.c_uint32),
        ("filter", C.c_int32), ("sharpen_percent", C.c_float), ("linear", C.c_int32),
        ("alpha_meaningful", C.c_int32), ("compose", C.c_int32), ("matte_bgra", C.c_uint8 * 4),
        ("color_matrix", C.c_void_p),
    ]


class OrientedResampleDesc(C.Structure):
    """struct ifb200_oriented_resample_desc"""
    _fields_ = [("draw", ResampleDesc), ("orientation", C.c_int32)]


class RowsResampleDesc(C.Structure):
    """struct ifb200_rows_resample_desc"""
    _fields_ = [("draw", ResampleDesc), ("format", C.c_int32)]


class RowsOrientedResampleDesc(C.Structure):
    """struct ifb200_rows_oriented_resample_desc"""
    _fields_ = [("draw", ResampleDesc), ("format", C.c_int32), ("orientation", C.c_int32)]


class RoundCornersDesc(C.Structure):
    """struct ifb200_round_corners_desc"""
    _fields_ = [
        ("px", C.c_void_p), ("w", C.c_uint32), ("h", C.c_uint32), ("stride", C.c_uint32),
        ("mode", C.c_int32), ("radius", C.c_float * 4), ("matte_bgra", C.c_uint8 * 4),
    ]


class CanvasDesc(C.Structure):
    """struct ifb200_canvas_desc"""
    _fields_ = [
        ("op", C.c_int32),
        ("px", C.c_void_p), ("w", C.c_uint32), ("h", C.c_uint32), ("stride", C.c_uint32), ("alpha_meaningful", C.c_int32),
        ("in_", C.c_void_p), ("in_w", C.c_uint32), ("in_h", C.c_uint32), ("in_stride", C.c_uint32), ("in_alpha_meaningful", C.c_int32),
        ("x1", C.c_uint32), ("y1", C.c_uint32), ("x2", C.c_uint32), ("y2", C.c_uint32), ("cw", C.c_uint32), ("ch", C.c_uint32),
        ("color_bgra", C.c_uint8 * 4),
    ]


class OrientDesc(C.Structure):
    """struct ifb200_orient_desc"""
    _fields_ = [
        ("in_", C.c_void_p), ("in_w", C.c_uint32), ("in_h", C.c_uint32), ("in_stride", C.c_uint32),
        ("out", C.c_void_p), ("out_stride", C.c_uint32), ("orientation", C.c_int32),
    ]


class ColorStep(C.Structure):
    """struct ifb200_color_step"""
    _fields_ = [("kind", C.c_int32), ("matrix", C.c_float * 25), ("threshold", C.c_float)]


class ColorDesc(C.Structure):
    """struct ifb200_color_desc"""
    _fields_ = [
        ("px", C.c_void_p), ("w", C.c_uint32), ("h", C.c_uint32), ("stride", C.c_uint32), ("alpha_meaningful", C.c_int32),
        ("steps", C.c_void_p), ("n_steps", C.c_uint32),
    ]


class WatermarkDesc(C.Structure):
    """struct ifb200_watermark_desc"""
    _fields_ = [("draw", ResampleDesc), ("opacity", C.c_float)]


class PixelConvertDesc(C.Structure):
    """struct ifb200_pixel_convert_desc"""
    _fields_ = [
        ("op", C.c_int32), ("src", C.c_void_p), ("src_stride", C.c_uint32), ("dst", C.c_void_p), ("dst_stride", C.c_uint32),
        ("w", C.c_uint32), ("h", C.c_uint32), ("opaque", C.c_int32),
    ]


class YcbcrDesc(C.Structure):
    """struct ifb200_ycbcr_desc"""
    _fields_ = [
        ("sampling", C.c_int32), ("y", C.c_void_p), ("y_stride", C.c_uint32), ("cb", C.c_void_p), ("cb_stride", C.c_uint32),
        ("cr", C.c_void_p), ("cr_stride", C.c_uint32), ("dst", C.c_void_p), ("dst_stride", C.c_uint32), ("w", C.c_uint32), ("h", C.c_uint32),
    ]


class BgraToYcbcrDesc(C.Structure):
    """struct ifb200_bgra_to_ycbcr_desc"""
    _fields_ = [
        ("sampling", C.c_int32), ("src", C.c_void_p), ("src_stride", C.c_uint32), ("y", C.c_void_p), ("y_stride", C.c_uint32),
        ("cb", C.c_void_p), ("cb_stride", C.c_uint32), ("cr", C.c_void_p), ("cr_stride", C.c_uint32), ("w", C.c_uint32), ("h", C.c_uint32),
        ("alpha_meaningful", C.c_int32), ("matte_bgra", C.c_uint8 * 4),
    ]


class SourceProfileDesc(C.Structure):
    """struct ifb200_source_profile"""
    _fields_ = [("kind", C.c_int32), ("icc", C.c_void_p), ("icc_len", C.c_size_t), ("gamma", C.c_double), ("chrm", C.c_double * 8),
                ("cicp", C.c_uint8 * 4)]


class ProfilePlan(C.Structure):
    """struct ifb200_profile_plan"""
    _fields_ = [("kind", C.c_int32), ("trc", (C.c_float * 256) * 3), ("m", (C.c_float * 3) * 3), ("gray", C.c_uint8 * 256)]


class ToSrgbDesc(C.Structure):
    """struct ifb200_to_srgb_desc"""
    _fields_ = [("format", C.c_int32), ("src", C.c_void_p), ("src_stride", C.c_uint32), ("dst", C.c_void_p), ("dst_stride", C.c_uint32),
                ("w", C.c_uint32), ("h", C.c_uint32), ("profile", C.c_void_p)]


class ProfiledResampleDesc(C.Structure):
    """struct ifb200_profiled_resample_desc"""
    _fields_ = [("draw", ResampleDesc), ("format", C.c_int32), ("orientation", C.c_int32), ("profile", C.c_void_p)]


class DetectContentDesc(C.Structure):
    """struct ifb200_detect_content_desc"""
    _fields_ = [("px", C.c_void_p), ("w", C.c_uint32), ("h", C.c_uint32), ("stride", C.c_uint32), ("alpha_meaningful", C.c_int32),
                ("threshold", C.c_uint32)]


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). imageflow_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    u32p, f32p, u8p = C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_uint8)
    L.ifb200_abi_version.restype = C.c_uint32
    L.ifb200_status_name.argtypes = [C.c_int]
    L.ifb200_status_name.restype = C.c_char_p
    L.ifb200_device_count.restype = C.c_int
    L.ifb200_weights.argtypes = [C.c_int, C.c_double, C.c_int, C.c_float, C.c_uint32, C.c_uint32, u32p, u32p, u32p, f32p, C.c_size_t]
    L.ifb200_weights.restype = C.c_int
    L.ifb200_byte_to_float_table.argtypes = [C.c_int, f32p]
    L.ifb200_byte_to_float_table.restype = None
    L.ifb200_linear_to_srgb_table.argtypes = [u8p]
    L.ifb200_linear_to_srgb_table.restype = None
    L.ifb200_color_filter_matrix.argtypes = [C.c_int, C.c_float, f32p]
    L.ifb200_color_filter_matrix.restype = C.c_int
    L.ifb200_plan_probe.argtypes = [C.POINTER(ResampleDesc), C.c_size_t, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_uint64),
                                    C.POINTER(C.c_uint64), C.c_char_p, C.c_size_t]
    L.ifb200_plan_probe.restype = C.c_int
    L.ifb200_scale_and_render.argtypes = [C.POINTER(ResampleDesc), C.c_char_p, C.c_size_t]
    L.ifb200_scale_and_render.restype = C.c_int
    L.ifb200_scale_and_render_many.argtypes = [C.POINTER(ResampleDesc), C.c_size_t, C.c_char_p, C.c_size_t]
    L.ifb200_scale_and_render_many.restype = C.c_int
    L.ifb200_color_matrix_bgra8.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, f32p, C.c_char_p, C.c_size_t]
    L.ifb200_color_matrix_bgra8.restype = C.c_int
    L.ifb200_apply_matte_bgra8.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, u8p, C.c_int, C.c_char_p, C.c_size_t]
    L.ifb200_apply_matte_bgra8.restype = C.c_int
    L.ifb200_batch_apply_matte.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, u8p, C.c_int, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_apply_matte.restype = C.c_int
    L.ifb200_transpose_bgra8.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_char_p, C.c_size_t]
    L.ifb200_transpose_bgra8.restype = C.c_int
    for f in (L.ifb200_flip_vertical_bgra8, L.ifb200_flip_horizontal_bgra8):
        f.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_char_p, C.c_size_t]
        f.restype = C.c_int
    L.ifb200_white_balance_srgb_bgra8.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, C.c_char_p, C.c_size_t]
    L.ifb200_white_balance_srgb_bgra8.restype = C.c_int
    u32p = C.POINTER(C.c_uint32)
    L.ifb200_detect_content_bgra8.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, u32p, C.c_char_p, C.c_size_t]
    L.ifb200_detect_content_bgra8.restype = C.c_int
    L.ifb200_batch_detect_content.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, u32p, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_detect_content.restype = C.c_int
    L.ifb200_batch_whitespace_codes.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_int, C.c_uint32, C.c_void_p, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_whitespace_codes.restype = C.c_int
    L.ifb200_detect_content_from_codes.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, u32p, C.POINTER(C.c_uint64)]
    L.ifb200_detect_content_from_codes.restype = C.c_int
    L.ifb200_batch_detect_content_many.argtypes = [C.c_void_p, C.POINTER(DetectContentDesc), C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                                   C.c_char_p, C.c_size_t]
    L.ifb200_batch_detect_content_many.restype = C.c_int
    L.ifb200_batch_white_balance.argtypes =[C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_white_balance.restype = C.c_int
    L.ifb200_batch_transpose.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_transpose.restype = C.c_int
    for f in (L.ifb200_batch_flip_vertical, L.ifb200_batch_flip_horizontal):
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_char_p, C.c_size_t]
        f.restype = C.c_int
    L.ifb200_batch_create.argtypes = [C.c_int, C.POINTER(C.c_void_p), C.c_char_p, C.c_size_t]
    L.ifb200_batch_create.restype = C.c_int
    L.ifb200_batch_enqueue.argtypes = [C.c_void_p, C.POINTER(ResampleDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_enqueue.restype = C.c_int
    L.ifb200_batch_enqueue_oriented.argtypes = [C.c_void_p, C.POINTER(OrientedResampleDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_enqueue_oriented.restype = C.c_int
    L.ifb200_batch_enqueue_rows.argtypes = [C.c_void_p, C.POINTER(RowsResampleDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_enqueue_rows.restype = C.c_int
    L.ifb200_batch_enqueue_rows_oriented.argtypes = [C.c_void_p, C.POINTER(RowsOrientedResampleDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_enqueue_rows_oriented.restype = C.c_int
    L.ifb200_batch_color_matrix.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, f32p, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_color_matrix.restype = C.c_int
    L.ifb200_batch_sync.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_sync.restype = C.c_int
    L.ifb200_batch_destroy.argtypes = [C.c_void_p]
    L.ifb200_batch_destroy.restype = None
    L.ifb200_batch_host_profile.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.c_int]
    L.ifb200_batch_host_profile.restype = C.c_int
    L.ifb200_batch_set_option.argtypes = [C.c_void_p, C.c_int, C.c_int64]
    L.ifb200_batch_set_option.restype = C.c_int
    for f in ("ifb200_batch_kernel_launches", "ifb200_batch_fused_jobs", "ifb200_batch_generic_jobs", "ifb200_batch_tile_jobs"):
        getattr(L, f).argtypes = [C.c_void_p]
        getattr(L, f).restype = C.c_uint64
    L.ifb200_block_scale_u8.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_char_p, C.c_size_t]
    L.ifb200_block_scale_u8.restype = C.c_int
    L.ifb200_batch_block_scale.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_block_scale.restype = C.c_int
    L.ifb200_round_corners_bgra8.argtypes = [C.POINTER(RoundCornersDesc), C.c_char_p, C.c_size_t]
    L.ifb200_round_corners_bgra8.restype = C.c_int
    L.ifb200_batch_round_corners.argtypes = [C.c_void_p, C.POINTER(RoundCornersDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_round_corners.restype = C.c_int
    L.ifb200_batch_canvas.argtypes = [C.c_void_p, C.POINTER(CanvasDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_canvas.restype = C.c_int
    L.ifb200_batch_orient.argtypes = [C.c_void_p, C.POINTER(OrientDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_orient.restype = C.c_int
    L.ifb200_batch_color_chain.argtypes = [C.c_void_p, C.POINTER(ColorDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_color_chain.restype = C.c_int
    L.ifb200_batch_watermark.argtypes = [C.c_void_p, C.POINTER(WatermarkDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_watermark.restype = C.c_int
    L.ifb200_batch_pixel_convert.argtypes = [C.c_void_p, C.POINTER(PixelConvertDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_pixel_convert.restype = C.c_int
    L.ifb200_batch_ycbcr_to_bgra.argtypes = [C.c_void_p, C.POINTER(YcbcrDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_ycbcr_to_bgra.restype = C.c_int
    L.ifb200_batch_bgra_to_ycbcr.argtypes = [C.c_void_p, C.POINTER(BgraToYcbcrDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_bgra_to_ycbcr.restype = C.c_int
    L.ifb200_batch_transform_to_srgb.argtypes = [C.c_void_p, C.POINTER(ToSrgbDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_transform_to_srgb.restype = C.c_int
    L.ifb200_batch_enqueue_profiled.argtypes = [C.c_void_p, C.POINTER(ProfiledResampleDesc), C.c_size_t, C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_enqueue_profiled.restype = C.c_int
    L.ifb200_source_profile_plan.argtypes = [C.POINTER(SourceProfileDesc), C.POINTER(ProfilePlan), C.c_char_p, C.c_size_t]
    L.ifb200_source_profile_plan.restype = C.c_int
    L.ifb200_batch_ring_status.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    L.ifb200_batch_ring_status.restype = C.c_int
    _lib = L
    return L
