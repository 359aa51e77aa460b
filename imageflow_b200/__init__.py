"""imageflow_b200 -- H100-native stand-in for imageflow's BGRA resample hot path.

Host-side mirror of the reference seam (paths relative to the imageflow checkout):
  graphics/scaling.rs:9-23      ScaleAndRenderParams, scale_and_render(input, canvas, &params)
  graphics/color_matrix.rs:5    window_bgra32_apply_color_matrix(window, matrix)
  graphics/weights.rs:45-78     Filter
  graphics/bitmaps.rs:156-160   BitmapCompositing
  graphics/blend.rs:6-59        apply_matte
  graphics/transpose.rs:95      bitmap_window_transpose;  graphics/flip.rs:10,25  flips
  flow/nodes/white_balance.rs   white_balance_srgb_mut (histogram.rs, area thresholds, byte maps)
  graphics/whitespace.rs:284    detect_content (code map on the GPU, the reference's window walk on the host)
  graphics/rounded_corners.rs:187  flow_bitmap_bgra_clear_around_rounded_corners, RoundCornersMode (imageflow_types)
  graphics/bitmaps.rs:1504,1570, graphics/copy_rect.rs:12  fill_rectangle, normalize_unused_alpha, copy_rectangle (Batch.canvas:
      FillRect, EnableTransparency, CopyRectToCanvas, ExpandCanvas; WatermarkRedDot, Region, RegionPercent as helpers)
  flow/nodes/rotate_flip_transpose.rs  ApplyOrientation, Rotate90/180/270, FlipH, FlipV, Transpose as one gather (Batch.orient,
      orientation_of; RIAPI's add_rotate / add_flip as riapi_rotate_steps / riapi_flip_steps)
  flow/nodes/color.rs, enable_transparency.rs, white_balance.rs  ColorMatrixSrgb, ColorFilterSrgb presets, EnableTransparency and
      WhiteBalanceHistogramAreaThresholdSrgb as one chain per frame (Batch.color_chain; RIAPI's s.* / a.balancewhite as riapi_color_steps)
  flow/nodes/watermark.rs, imageflow_riapi ir4/layout.rs + sizing.rs  Watermark: its layout (watermark_layout, process_constraint) and
      every frame's composite from one resample per distinct watermark (Batch.watermark; RIAPI's placement as riapi_watermark_placement)
  graphics/swizzle.rs, bitmaps.rs:1284-1345  rgb_to_bgra, copy_swap_br, gray_to_bgra, gray_alpha_to_bgra, to_vec_rgb: decoder rows into
      BGRA and encoder rows out of it, batched (Batch.pixel_convert over PixelRows; Batch.to_bgra / from_bgra for one tensor)
  c_components/lib/codecs_jpeg_idct_fast.c  flow_scale_spatial[_srgb]_NxN (decode-time JPEG block scalers)
All arithmetic runs in hand-written sm_90a kernels inside libifb200.so (include/ifb200.h);
this package only marshals arguments.  Nothing here imports the CPU oracle.
"""
from .graphics import (Batch, apply_matte, BitmapCompositing, BitmapWindow, ErrorKind, Filter, FlowError, ScaleAndRenderParams,
                       WorkingFloatspace, color_filter_matrix, device_count, plan_probe, populate_weights, scale_and_render, scale_and_render_many,
                       window_bgra32_apply_color_matrix, bitmap_window_transpose, flow_bitmap_bgra_flip_vertical_safe,
                       flow_bitmap_bgra_flip_horizontal_safe, white_balance_srgb_mut, detect_content, detect_content_from_codes, flow_scale_spatial,
                       RoundCornersMode, flow_bitmap_bgra_clear_around_rounded_corners,
                       FillRect, CopyRectToCanvas, ExpandCanvas, EnableTransparency, new_canvas, watermark_red_dot, region, region_percent,
                       ApplyOrientation, Rotate90, Rotate180, Rotate270, FlipH, FlipV, Transpose, orientation_of, riapi_rotate_steps,
                       riapi_flip_steps, apply_orientation, ColorMatrixSrgb, ColorFilterSrgb, WhiteBalanceHistogramAreaThresholdSrgb,
                       riapi_color_steps, Watermark, WatermarkConstraintBox, WatermarkConstraintMode, ConstraintGravity, WatermarkDraw,
                       process_constraint, watermark_layout, riapi_watermark_placement, PixelRows, RgbToBgra, RgbaToBgra, GrayToBgra,
                       GrayAlphaToBgra, BgraToRgb, pixel_op_for)
from ._lib import LIB_PATH, ResampleDesc, lib

__all__ = [
    "Batch", "apply_matte", "BitmapCompositing", "BitmapWindow", "ErrorKind", "Filter", "FlowError", "ScaleAndRenderParams",
    "WorkingFloatspace", "color_filter_matrix", "device_count", "plan_probe", "populate_weights", "scale_and_render", "scale_and_render_many",
    "window_bgra32_apply_color_matrix", "bitmap_window_transpose", "flow_bitmap_bgra_flip_vertical_safe",
    "flow_bitmap_bgra_flip_horizontal_safe", "white_balance_srgb_mut", "detect_content", "detect_content_from_codes", "flow_scale_spatial",
    "RoundCornersMode", "flow_bitmap_bgra_clear_around_rounded_corners",
    "FillRect", "CopyRectToCanvas", "ExpandCanvas", "EnableTransparency", "new_canvas", "watermark_red_dot", "region", "region_percent",
    "ApplyOrientation", "Rotate90", "Rotate180", "Rotate270", "FlipH", "FlipV", "Transpose", "orientation_of", "riapi_rotate_steps",
    "riapi_flip_steps", "apply_orientation", "ColorMatrixSrgb", "ColorFilterSrgb", "WhiteBalanceHistogramAreaThresholdSrgb",
    "riapi_color_steps", "Watermark", "WatermarkConstraintBox", "WatermarkConstraintMode", "ConstraintGravity", "WatermarkDraw",
    "process_constraint", "watermark_layout", "riapi_watermark_placement", "PixelRows", "RgbToBgra", "RgbaToBgra", "GrayToBgra",
    "GrayAlphaToBgra", "BgraToRgb", "pixel_op_for", "LIB_PATH", "ResampleDesc", "lib",
]
