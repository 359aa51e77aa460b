/*
 * ifb200.h -- C ABI of the H100-native resample engine (libifb200.so).
 *
 * This is the drop-in boundary for ONE hot path of imazen/imageflow: the BGRA8
 * resample / composite / colour-matrix path behind
 *     imageflow_core::graphics::scaling::scale_and_render        (graphics/scaling.rs:19-90)
 *     imageflow_core::graphics::color_matrix::window_bgra32_apply_color_matrix (graphics/color_matrix.rs:5-28)
 * which the flow-graph executors DrawImageDef::render (flow/nodes/scale_render.rs:304-313) and
 * ColorMatrixSrgbMutDef::mutate (flow/nodes/color.rs:26-28) call.  (All paths relative to the
 * reference checkout; INTEGRATION.md shows the Rust `extern "C"` block that binds these symbols.)
 *
 * Plain pointers and sizes only; no C++/torch types.  Every function is thread-safe, never throws
 * or aborts across the boundary, never retains caller pointers after it returns (batch jobs: after
 * ifb200_batch_sync returns).  There is NO CPU fallback: without a usable CUDA device every compute
 * entry point fails with IFB200_ERR_NO_DEVICE.
 */
#ifndef IFB200_H
#define IFB200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define IFB200_ABI_VERSION_MAJOR 1
#define IFB200_ABI_VERSION_MINOR 2

/* Error codes.  1..3 map onto the imageflow ErrorKind values raised by scale_and_render
 * (scaling.rs:24-48,145,191,202,240); 10..12 onto WeightsError (weights.rs:494-504). */
enum ifb200_status {
    IFB200_OK = 0,
    IFB200_ERR_INVALID_ARGUMENT = 1,      /* ErrorKind::InvalidArgument  (scaling.rs:24-29,38-40) */
    IFB200_ERR_NOT_IMPLEMENTED = 2,       /* ErrorKind::MethodNotImplemented (scaling.rs:43-48)   */
    IFB200_ERR_INVALID_STATE = 3,         /* ErrorKind::InvalidState (scaling.rs:145,191,202,240) */
    IFB200_ERR_TOTAL_WEIGHT_ZERO = 10,    /* WeightsError::TotalWeightZero (weights.rs:755-757)   */
    IFB200_ERR_SOURCE_COUNT_TOO_LARGE = 11,
    IFB200_ERR_NO_PIXEL_INPUTS = 12,
    IFB200_ERR_BAD_FILTER = 13,
    IFB200_ERR_CAPACITY = 14,
    IFB200_ERR_NO_DEVICE = 20,            /* no CUDA device / driver: there is no CPU fallback    */
    IFB200_ERR_CUDA = 21,                 /* a CUDA runtime call failed; message has the detail   */
    IFB200_ERR_OUT_OF_MEMORY = 22
};

/* weights.rs:45-78 -- `Filter` repr(C) discriminants, used verbatim. */
enum ifb200_filter {
    IFB200_FILTER_ROBIDOUX_FAST = 1, IFB200_FILTER_ROBIDOUX = 2, IFB200_FILTER_ROBIDOUX_SHARP = 3,
    IFB200_FILTER_GINSENG = 4, IFB200_FILTER_GINSENG_SHARP = 5, IFB200_FILTER_LANCZOS = 6,
    IFB200_FILTER_LANCZOS_SHARP = 7, IFB200_FILTER_LANCZOS2 = 8, IFB200_FILTER_LANCZOS2_SHARP = 9,
    IFB200_FILTER_CUBIC_FAST = 10, IFB200_FILTER_CUBIC = 11, IFB200_FILTER_CUBIC_SHARP = 12,
    IFB200_FILTER_CATMULL_ROM = 13, IFB200_FILTER_MITCHELL = 14, IFB200_FILTER_CUBIC_BSPLINE = 15,
    IFB200_FILTER_HERMITE = 16, IFB200_FILTER_JINC = 17, IFB200_FILTER_RAW_LANCZOS3 = 18,
    IFB200_FILTER_RAW_LANCZOS3_SHARP = 19, IFB200_FILTER_RAW_LANCZOS2 = 20, IFB200_FILTER_RAW_LANCZOS2_SHARP = 21,
    IFB200_FILTER_TRIANGLE = 22, IFB200_FILTER_LINEAR = 23, IFB200_FILTER_BOX = 24,
    IFB200_FILTER_CATMULL_ROM_FAST = 25, IFB200_FILTER_CATMULL_ROM_FAST_SHARP = 26, IFB200_FILTER_FASTEST = 27,
    IFB200_FILTER_MITCHELL_FAST = 28, IFB200_FILTER_NCUBIC = 29, IFB200_FILTER_NCUBIC_SHARP = 30,
    IFB200_FILTER_LEGACY_IDCT = 31
};

/* graphics/bitmaps.rs:156-160 BitmapCompositing */
enum ifb200_compose { IFB200_REPLACE_SELF = 0, IFB200_BLEND_WITH_SELF = 1, IFB200_BLEND_WITH_MATTE = 2 };
/* weights.rs:16-23 LobeRatio */
enum ifb200_lobe { IFB200_LOBE_NATURAL = 0, IFB200_LOBE_EXACT = 1, IFB200_LOBE_SHARPEN_PERCENT = 2 };

/* One scale_and_render call: (input window, canvas window, ScaleAndRenderParams) -- scaling.rs:9-23. */
typedef struct ifb200_resample_desc {
    const uint8_t* in;  uint32_t in_w, in_h, in_stride;   /* BGRA8 sRGB, straight alpha; stride in bytes (bitmaps.rs:712-740) */
    uint8_t* canvas;    uint32_t cv_w, cv_h, cv_stride;   /* the canvas BEFORE cropping to (x,y,w,h) (scaling.rs:30-41)      */
    uint32_t x, y, w, h;                                   /* ScaleAndRenderParams.x/y/w/h                                    */
    int32_t  filter;                                       /* enum ifb200_filter (ScaleAndRenderParams.interpolation_filter)   */
    float    sharpen_percent;                              /* sharpen_percent_goal; <= 0 means off (scaling.rs:104-106)       */
    int32_t  linear;                                       /* 1 = WorkingFloatspace::LinearRGB, 0 = StandardRGB (scaling.rs:52) */
    int32_t  alpha_meaningful;                             /* input.info().alpha_meaningful() (scaling.rs:51)                 */
    int32_t  compose;                                      /* enum ifb200_compose = canvas.info().compose() (scaling.rs:50)   */
    uint8_t  matte_bgra[4];                                /* BlendWithMatte colour as to_bgra8() (scaling.rs:67)            */
    const float* color_matrix;                             /* optional fused ColorMatrixSrgb (row-major [5][5]) applied to the
                                                              destination rect after the render; NULL = none (color_matrix.rs) */
} ifb200_resample_desc;

/* ---- library / device ---------------------------------------------------------------------- */
uint32_t    ifb200_abi_version(void);                      /* (major << 16) | minor */
/* Device of the host-buffer (drop-in) calls made by threads that have not made one yet (each calling thread keeps its own context on
 * the device that was selected when it made its first call).  Default: the IFB200_DEVICE environment variable, else device 0. */
int         ifb200_set_dropin_device(int device);
const char* ifb200_status_name(int status);
int         ifb200_device_count(void);                     /* 0 when no CUDA device / driver is usable */

/* ---- host-side specification helpers (no GPU needed) ----------------------------------------
 * populate_weights (weights.rs:681-788) for one axis. left/right hold out_size entries, offsets
 * out_size+1 (prefix offsets into weights[]).  kernel_width_scale = set_kernel_width_scale factor
 * (weights.rs:156-158), lobe_* = LobeRatio (weights.rs:16-40). */
int ifb200_weights(int filter, double kernel_width_scale, int lobe_mode, float lobe_value,
                   uint32_t out_size, uint32_t in_size,
                   uint32_t* left, uint32_t* right, uint32_t* offsets,
                   float* weights, size_t weights_cap);
/* ColorContext::byte_to_float (color.rs:23-48) and LINEAR_TO_SRGB_LUT (lut.rs:14) as uploaded to the device */
void ifb200_byte_to_float_table(int linear, float out[256]);
void ifb200_linear_to_srgb_table(uint8_t out[16384]);
/* ColorFilterSrgb presets (flow/nodes/color.rs:86-225): 0 sepia, 1 grayscale_ntsc, 2 grayscale_flat,
 * 3 grayscale_bt709, 4 grayscale_ry, 5 invert, 6 alpha(p), 7 contrast(p), 8 brightness(p), 9 saturation(p) */
int  ifb200_color_filter_matrix(int which, float p, float out[25]);
/* detect_content with a HOST bitmap (drop-in for graphics/whitespace.rs:284); and its host half alone: the window walk over a
 * w*h code map (layout: imageflow_b200/csrc/ifb_whitespace.h), no CUDA call -- `centres` (optional) = pixels visited. */
int  ifb200_detect_content_bgra8(const uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, int alpha_meaningful, uint32_t threshold,
                                 uint32_t rect[4], char* err, size_t err_cap);
int  ifb200_detect_content_from_codes(const uint8_t* codes, uint32_t w, uint32_t h, uint32_t rect[4], uint64_t* centres);
/* Host-side cost of preparing kernel tables (benchmarks of mixed workloads, where every geometry is new): builds the plans of
   descs[0..n) -- only in_w, in_h, w, h, filter, sharpen_percent are read -- on `threads` host threads and discards them.
   No CUDA call.  *table_hash (optional) = a hash of every table built, independent of the thread count. */
int  ifb200_plan_probe(const ifb200_resample_desc* descs, size_t n, int threads, double* seconds, uint64_t* table_bytes,
                       uint64_t* table_hash, char* err, size_t err_cap);

/* The streaming ring kernel's host tables for one geometry (only in_w, in_h, w, h, filter, sharpen_percent are read), as they
   would be uploaded (alpha_meaningful selects the 3- or 4-channel kernel variant's strip width): call with buf = NULL for the size.  info->ok == 0: the geometry does not run on the ring kernel.
   Layout: imageflow_b200/csrc/ifb_hv_kernel.cuh (HvStripDev, HvBandDev, HvPlanDev).  No CUDA call. */
typedef struct ifb200_hv_plan_info {
    int32_t ok, av, n_strips, n_bands, cap_px /* weight records per strip in hw; hdone has cap_px + 64 bytes per strip */, avp;
    uint64_t o_strips, o_hw, o_hdone, o_vw, o_vdone, o_bands, total;
} ifb200_hv_plan_info;
int  ifb200_hv_plan_tables(const ifb200_resample_desc* d, int strip_cols, int n_band_pairs, ifb200_hv_plan_info* info, uint8_t* buf, size_t cap,
                           char* err, size_t err_cap);

/* ---- drop-in calls: HOST buffers, synchronous (what the Rust adapter calls) ------------------
 * Replaces the bodies of scaling.rs:93-251 (resize_to_canvas / resize_with_matte /
 * resize_and_composite).  err (may be NULL) receives a NUL-terminated message on failure. */
int ifb200_scale_and_render(const ifb200_resample_desc* desc, char* err, size_t err_cap);
/* The same for n independent calls (e.g. the DrawImageExact nodes of one graph, or export_4_sizes): identical
 * results, but uploads, kernels and downloads of consecutive jobs are pipelined on several CUDA streams.
 * Jobs must not alias each other's canvases.  Argument errors are reported before any job runs. */
int ifb200_scale_and_render_many(const ifb200_resample_desc* descs, size_t n, char* err, size_t err_cap);
/* Replaces color_matrix.rs:5-28 (in place). */
int ifb200_color_matrix_bgra8(uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, const float m[25],
                              char* err, size_t err_cap);

/* Replaces Bitmap::apply_matte (graphics/blend.rs:6-59), the encoder-side flatten over a solid colour (in place,
 * linear light).  No-op unless alpha is meaningful (blend.rs:10-13).  [SURVEY.md section 8(f), item 2] */
int ifb200_apply_matte_bgra8(uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, const uint8_t matte_bgra[4],
                             int alpha_meaningful, char* err, size_t err_cap);

/* Replaces graphics::transpose::bitmap_window_transpose (graphics/transpose.rs:95-121; checks of :46-79):
 * to[x][y] = from[y][x] for a w x h BGRA8 window; `to` is h pixels wide and w rows tall.  Strides in bytes.
 * [SURVEY.md section 8(f), item 3] */
int ifb200_transpose_bgra8(const uint8_t* from, uint32_t from_stride, uint32_t w, uint32_t h, uint8_t* to, uint32_t to_stride,
                           char* err, size_t err_cap);
/* Replace flow_bitmap_bgra_flip_vertical_safe / flow_bitmap_bgra_flip_horizontal_safe (graphics/flip.rs:10-22, 25-39), in place. */
int ifb200_flip_vertical_bgra8(uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, char* err, size_t err_cap);
int ifb200_flip_horizontal_bgra8(uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, char* err, size_t err_cap);

/* Replaces the work of WhiteBalanceSrgbMutDef::mutate (flow/nodes/white_balance.rs:93-121): per-channel histograms
 * (graphics/histogram.rs:7-20), area thresholds and byte maps (white_balance.rs:14-48), in-place remap of B, G, R (:50-67).
 * threshold < 0 = None (0.006).  [SURVEY.md section 8(f), item 4] */
int ifb200_white_balance_srgb_bgra8(uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, float threshold, char* err, size_t err_cap);

/* Replaces flow_scale_spatial[_srgb]_{n}x{n} (c_components/lib/codecs_jpeg_idct_fast.c:302-4428; libjpeg hook codec_jpeg_wrapper.c:232-340,
 * enabled by JpegDownscaleHints, mozjpeg_decoder.rs:593-611) for a whole plane of samples: every 8x8 block of `in` (blocks_x x blocks_y
 * blocks, row stride in_stride bytes) becomes the n x n block at (bx*n, by*n) of `out`; n = 1..7; srgb != 0 = the linear-light variants.
 * Bit-identical to the reference functions (integer arithmetic, the reference's own weight and table literals).
 * [SURVEY.md section 8(f), item 1] */
int ifb200_block_scale_u8(const uint8_t* in, uint32_t in_stride, uint32_t blocks_x, uint32_t blocks_y, uint8_t* out, uint32_t out_stride,
                          int n, int srgb, char* err, size_t err_cap);

/* Replaces flow_bitmap_bgra_clear_around_rounded_corners (graphics/rounded_corners.rs:187-346), the op behind RoundImageCorners /
 * s.roundcorners= (flow/nodes/round_corners.rs:62-84): pixels outside the rounded corners become the matte, the arcs are
 * anti-aliased over it in linear light, in place.  [SURVEY.md section 8(f), item 5]
 * Modes: imageflow_types RoundCornersMode (lib.rs:1257-1268), in declaration order.  Radii that the reference clamps, ceils or
 * truncates (negative, NaN, infinite, oversized) behave exactly as they do there; they are not errors. */
enum ifb200_corners_mode { IFB200_CORNERS_PERCENTAGE = 0, IFB200_CORNERS_PIXELS = 1, IFB200_CORNERS_CIRCLE = 2,
                           IFB200_CORNERS_PERCENTAGE_CUSTOM = 3, IFB200_CORNERS_PIXELS_CUSTOM = 4 };
typedef struct ifb200_round_corners_desc {
    uint8_t* px; uint32_t w, h, stride;   /* BGRA8 window, in place; stride in bytes */
    int32_t  mode;                        /* enum ifb200_corners_mode */
    float    radius[4];                   /* top_left, top_right, bottom_right, bottom_left (the field order of
                                             RoundCornersMode::*Custom); [0] alone for PERCENTAGE / PIXELS; unused for CIRCLE */
    uint8_t  matte_bgra[4];               /* background_color.to_color_32().to_bgra8() */
} ifb200_round_corners_desc;
/* HOST window, synchronous.  Only the pixels the op can touch travel to the GPU and back (a few rectangles at the corners; rectangles
 * that are only filled with the matte are not uploaded). */
int ifb200_round_corners_bgra8(const ifb200_round_corners_desc* d, char* err, size_t err_cap);

/* The canvas layer of a flow graph, on BGRA8 windows (alpha_meaningful = 1 is the reference's Bgra32, 0 its Bgr32):
 *   FILL_RECT        BitmapWindowMut::fill_rectangle(color, x1, y1, x2, y2) (graphics/bitmaps.rs:1504-1562): FillRect, WatermarkRedDot.
 *                    x2 == x1 or y2 == y1 is a no-op (even out of bounds); otherwise the rectangle must lie inside the window.
 *   COPY_RECT        copy_rectangle(in, canvas, x1, y1, x2, y2, cw, ch) (graphics/copy_rect.rs:12-97): CopyRectToCanvas.  A Bgr32
 *                    canvas under a Bgra32 input first gets A = 255 over its whole window; a Bgr32 input under a Bgra32 canvas gets
 *                    A = 255 over its whole window, in place.  Then the rows are copied as raw bytes (stride padding is not).
 *   EXPAND           ExpandCanvas { left = x1, top = y1, right = x2, bottom = y2, color } (flow/nodes/clone_crop_fill_expand.rs:224-260)
 *                    into the caller's new canvas px (w = in_w + left + right, h = in_h + top + bottom): the border becomes color,
 *                    the interior the input, as COPY_RECT into a Bgr32 (color opaque, a == 255, and input Bgr32) or Bgra32 canvas.
 *                    The descriptor's alpha_meaningful is not read: that format rule decides it.
 *   NORMALIZE_ALPHA  normalize_unused_alpha (graphics/bitmaps.rs:1564-1576): A = 255 over the window unless alpha_meaningful.
 * Each pixel is written once (EXPAND fills only the border).  Bitmap metadata checks (BGRA only, BlendWithMatte sub-rectangles,
 * EnableTransparency on a Bgra32 bitmap) stay with the caller.  24-bit inputs are not supported. */
enum ifb200_canvas_op { IFB200_CANVAS_FILL_RECT = 0, IFB200_CANVAS_COPY_RECT = 1, IFB200_CANVAS_EXPAND = 2, IFB200_CANVAS_NORMALIZE_ALPHA = 3 };
typedef struct ifb200_canvas_desc {
    int32_t  op;                                               /* enum ifb200_canvas_op */
    uint8_t* px; uint32_t w, h, stride; int32_t alpha_meaningful;             /* the window written: FILL / NORMALIZE target, COPY
                                                                                 canvas, EXPAND's new canvas; stride in bytes   */
    uint8_t* in; uint32_t in_w, in_h, in_stride; int32_t in_alpha_meaningful; /* COPY / EXPAND source; not const: a Bgr32 input
                                                                                 under a Bgra32 canvas gets A = 255 in place     */
    uint32_t x1, y1, x2, y2;   /* FILL: x, y, x2, y2.  COPY: from_x, from_y, to_x, to_y.  EXPAND: left, top, right, bottom */
    uint32_t cw, ch;           /* COPY: w, h */
    uint8_t  color_bgra[4];    /* FILL / EXPAND: Color::to_bgra8() */
} ifb200_canvas_desc;

/* One orientation job: ApplyOrientation { flag } (flow/nodes/rotate_flip_transpose.rs:50-66) and every chain of Rotate90 / 180 /
 * 270, FlipH, FlipV and Transpose, which compose into one of the eight EXIF orientations.  With the input window w x h, the output
 * is w x h for 1..4 and h x w for 5..8, and out(x, y) = in(...) with
 *   1 (x, y)   2 (w-1-x, y)   3 (w-1-x, h-1-y)   4 (x, h-1-y)   5 (y, x)   6 (y, h-1-x)   7 (w-1-y, h-1-x)   8 (w-1-y, x)
 * Pixels move as raw 4-byte words, alpha included.  Any flag other than 2..8 is the identity, as the reference's `_ => vec![]`.
 * out == in (same pointer and stride) is in place, allowed for 1..4 only (the reference panics on an in-place transpose,
 * :158-160); otherwise the input and output byte spans must not overlap.  A job of zero area is skipped unchecked. */
typedef struct ifb200_orient_desc {
    const uint8_t* in;  uint32_t in_w, in_h, in_stride;   /* BGRA8 window; stride in bytes */
    uint8_t*       out; uint32_t out_stride;              /* in_w x in_h for 1..4, in_h x in_w for 5..8; may equal `in` for 1..4 */
    int32_t        orientation;                           /* EXIF flag; values other than 2..8 are the identity */
} ifb200_orient_desc;

/* One colour chain: the photometric nodes of a flow graph applied in order to one BGRA8 window, in place, byte for byte as the
 * reference runs them node by node (each node requantises to bytes, so a chain is not one matrix):
 *   MATRIX               ColorMatrixSrgb { matrix } = window_bgra32_apply_color_matrix (graphics/color_matrix.rs:5-28): every output
 *                        channel from the pixel's original four bytes, the sum left to right in f32 (bias m[4][c] * 255 last), then
 *                        uchar_clamp_ff.  NaN and infinite coefficients are not errors: they compute what the reference computes.
 *                        ColorFilterSrgb presets are matrices (ifb200_color_filter_matrix); Alpha is ENABLE_TRANSPARENCY + MATRIX.
 *   ENABLE_TRANSPARENCY  the EnableTransparency node (flow/nodes/enable_transparency.rs:27-33): on a Bgr32 window A = 255 and the job
 *                        is Bgra32 from then on; on Bgra32 nothing (the node deletes itself there).
 *   WHITE_BALANCE        WhiteBalanceHistogramAreaThresholdSrgb { threshold } (flow/nodes/white_balance.rs:93-121): R, G, B histograms
 *                        of the whole window as the chain has left it at that step, area thresholds and byte maps in f64, R, G, B
 *                        remapped, alpha untouched.  threshold < 0 = None (0.006), NaN refused.  At most one per job.
 * A job with no steps or no pixels is skipped unchecked.  Only pixels are written: the bitmap metadata the nodes change stays with the
 * caller (BlendWithSelf after any MATRIX, color.rs:29; Bgra32 + BlendWithSelf after ENABLE_TRANSPARENCY on Bgr32). */
enum ifb200_color_step_kind { IFB200_COLOR_MATRIX = 0, IFB200_COLOR_ENABLE_TRANSPARENCY = 1, IFB200_COLOR_WHITE_BALANCE = 2 };
#define IFB200_COLOR_MAX_STEPS 16          /* steps per job; RIAPI's s.* / a.balancewhite keys make at most 8 */
typedef struct ifb200_color_step {
    int32_t kind;                          /* enum ifb200_color_step_kind */
    float   matrix[25];                    /* MATRIX: row-major [5][5] exactly as color_matrix.rs reads it (m[k][c]: input k, output c) */
    float   threshold;                     /* WHITE_BALANCE: < 0 = None (0.006); NaN refused */
} ifb200_color_step;
typedef struct ifb200_color_desc {
    uint8_t* px; uint32_t w, h, stride;    /* BGRA8 window, in place; stride in bytes */
    int32_t  alpha_meaningful;             /* the window's format going in: Bgra32 (1) or Bgr32 (0) */
    const ifb200_color_step* steps;        /* HOST array of n_steps steps, applied in order; read before the call returns */
    uint32_t n_steps;
} ifb200_color_desc;

/* One watermark composite: the work of the nodes WatermarkDef::expand (flow/nodes/watermark.rs:96-205) leaves behind for one frame, after
 * the caller has done the layout (crop, x, y, w, h, filter):
 *   draw     the DrawImageExact of the watermark onto the frame.  draw.in is the watermark window AFTER the layout's crop (a sub-window
 *            at any 4-byte offset), draw.canvas the frame, draw.alpha_meaningful the watermark's format, draw.compose the frame's
 *            compositing mode going in: the library applies the Compose rule itself (ReplaceSelf is drawn as BlendWithSelf,
 *            scale_render.rs:282-284; BlendWithSelf and BlendWithMatte stay).  color_matrix must be NULL.
 *   opacity  Watermark.opacity.unwrap_or(1) as given: clamped to [0, 1] and, when < 1, applied as ColorFilterSrgb::Alpha (EnableTransparency
 *            + the alpha matrix) to a private copy of the window before the draw (watermark.rs:166-172); NaN and >= 1 mean no opacity step.
 * The caller's watermark is never written.  Afterwards the frame is BlendWithSelf (scale_render.rs:314): the caller sets that. */
typedef struct ifb200_watermark_desc {
    ifb200_resample_desc draw;
    float opacity;
} ifb200_watermark_desc;

/* One resample of an oriented frame: scale_and_render(orient(draw.in, orientation), canvas, params), byte for byte, without the
 * oriented frame ever being written -- the decode -> ApplyOrientation -> DrawImageExact chain of a photo with an EXIF orientation
 * (and RIAPI's srotate / sflip folded into the flag with the orientation of ifb200_orient_desc).
 *   draw         draw.in / in_w / in_h / in_stride: the SOURCE window as stored (not rotated); the resample sees orient(draw.in,
 *                orientation): in_w x in_h for 1..4, in_h x in_w for 5..8.  Every other field as in ifb200_batch_enqueue.
 *   orientation  EXIF flag, the closed form of ifb200_orient_desc; values other than 2..8 are the identity.
 * The arithmetic is that of the resample of the materialised oriented frame: the H chain ascends over oriented columns and the V
 * chain over oriented rows (descending source coordinates along a reversed axis; along a source column for 5..8). */
typedef struct ifb200_oriented_resample_desc {
    ifb200_resample_desc draw;
    int32_t orientation;
} ifb200_oriented_resample_desc;

/* One pixel-format conversion at the edge of a flow graph: the row swizzles of graphics/swizzle.rs:8-45 that the decoders call into
 * BGRA (image_png_decoder.rs:156-193, jpeg_decoder.rs:103-129) and the RGB rows the encoders take out of it (bitmaps.rs:1284-1345).
 * Per pixel, source bytes -> destination bytes:
 *   RGB24_TO_BGRA       rgb_to_bgra          (r, g, b)    -> (b, g, r, 255)
 *   RGBA_TO_BGRA        copy_swap_br         (r, g, b, a) -> (b, g, r, a); symmetric, so also BGRA -> RGBA
 *   GRAY_TO_BGRA        gray_to_bgra         (v)          -> (v, v, v, 255)
 *   GRAY_ALPHA_TO_BGRA  gray_alpha_to_bgra   (v, a)       -> (v, v, v, a)
 *   BGRA_TO_RGB24       to_vec_rgb           (b, g, r, a) -> (r, g, b): alpha dropped, no matte
 * opaque != 0 writes 255 into every alpha byte of a 4-byte output (the encoders' swap-then-fill-alpha, zen_encoder.rs:585-603, in one
 * pass); BGRA_TO_RGB24 has none and ignores it.  Fill-alpha alone is IFB200_CANVAS_NORMALIZE_ALPHA.  RGBA_TO_BGRA may run in place
 * (src == dst with the same stride: swap_br_inplace); any other overlap of the source and destination byte spans is refused.  Strides
 * must hold a row; a 4-byte output needs a 4-byte aligned dst and dst_stride, while 1-, 2- and 3-byte rows may start at any byte.  A job
 * of zero area is skipped unchecked.  Planar (CHW), 16-bit and indexed sources are not covered. */
enum ifb200_pixel_op { IFB200_PIXEL_RGB24_TO_BGRA = 0, IFB200_PIXEL_RGBA_TO_BGRA = 1, IFB200_PIXEL_GRAY_TO_BGRA = 2,
                       IFB200_PIXEL_GRAY_ALPHA_TO_BGRA = 3, IFB200_PIXEL_BGRA_TO_RGB24 = 4 };
typedef struct ifb200_pixel_convert_desc {
    int32_t        op;                      /* enum ifb200_pixel_op */
    const uint8_t* src; uint32_t src_stride;   /* w x h source window; stride in bytes */
    uint8_t*       dst; uint32_t dst_stride;   /* w x h destination window; may equal src for RGBA_TO_BGRA */
    uint32_t       w, h;
    int32_t        opaque;                  /* != 0: alpha = 255 in a 4-byte output */
} ifb200_pixel_convert_desc;

/* One JPEG frame's colour stage: the Y, Cb and Cr planes a GPU JPEG decoder hands over (nvJPEG's NVJPEG_OUTPUT_YUV, at the file's
 * chroma subsampling) into a BGRA frame, byte for byte as libjpeg-turbo decodes into JCS_EXT_BGRA with its defaults (the reference's
 * mozjpeg decoder, codecs/mozjpeg_decoder.rs): fancy chroma upsampling, then the fixed-point YCbCr -> RGB tables.  Per pixel, with
 * y, cb, cr the samples after upsampling:
 *   R = clamp(y + ((91881 (cr - 128) + 32768) >> 16))                      FIX(1.40200)
 *   G = clamp(y + ((-22554 (cb - 128) + 32768 - 46802 (cr - 128)) >> 16))  FIX(0.34414), FIX(0.71414)
 *   B = clamp(y + ((116130 (cb - 128) + 32768) >> 16))                     FIX(1.77200)
 * with >> arithmetic and clamp to 0..255; alpha is 255.  Upsampling, neighbours clamped to the plane (edge rows and columns repeated):
 *   444  none: the chroma planes are w x h.
 *   422  chroma ceil(w/2) x h; output column 2i = (3 c[i] + c[i-1] + 1) >> 2, 2i+1 = (3 c[i] + c[i+1] + 2) >> 2 (h2v1_fancy_upsample).
 *   420  chroma ceil(w/2) x ceil(h/2); column sums s = 3 c[j] + c[j-1] for output row 2j and 3 c[j] + c[j+1] for row 2j+1, then
 *        output column 2i = (3 s[i] + s[i-1] + 8) >> 4, 2i+1 = (3 s[i] + s[i+1] + 7) >> 4 (h2v2_fancy_upsample).
 * A chroma plane one or two columns wide is replicated instead (libjpeg-turbo runs the fancy forms only above two columns).  Planes
 * may sit at any byte address with any pitch that holds a row; the destination is 4-byte aligned.  A grayscale JPEG needs none of
 * this: its one plane is Gray8 rows, and IFB200_PIXEL_GRAY_TO_BGRA is libjpeg's gray -> BGRA.  4:4:0, 4:1:1, CMYK / YCCK and
 * Adobe-transform-0 (RGB-coded) JPEGs are not covered. */
enum ifb200_ycbcr_sampling { IFB200_YCBCR_444 = 0, IFB200_YCBCR_422 = 1, IFB200_YCBCR_420 = 2 };
typedef struct ifb200_ycbcr_desc {
    int32_t        sampling;                /* enum ifb200_ycbcr_sampling */
    const uint8_t* y;  uint32_t y_stride;   /* w x h luma */
    const uint8_t* cb; uint32_t cb_stride;  /* chroma planes at the sampling's size; each plane has its own pitch */
    const uint8_t* cr; uint32_t cr_stride;
    uint8_t*       dst; uint32_t dst_stride;   /* w x h BGRA: 4-byte aligned pointer and stride */
    uint32_t       w, h;
} ifb200_ycbcr_desc;

/* One JPEG frame's encoder colour stage, the way back: a BGRA frame into the Y, Cb and Cr planes a GPU JPEG encoder takes (nvJPEG's
 * nvjpegEncodeYUV), byte for byte what libjpeg-turbo's compressor holds before its DCT when it is fed apply_matte(src) as JCS_EXT_BGRA
 * with jpeg_set_defaults (no smoothing) and the given sampling -- the reference's MozjpegEncoder::write_frame (codecs/mozjpeg.rs).
 *   Matte   when alpha_meaningful != 0, each pixel is first flattened over matte_bgra exactly as ifb200_batch_apply_matte does
 *           (graphics/blend.rs, linear light); the source is never written.  Alpha is then ignored, as libjpeg ignores it.
 *   Colour  jccolor.c rgb_ycc_convert, >> arithmetic, results always in 0..255:
 *             Y  = (19595 R + 38470 G + 7471 B + 32768) >> 16
 *             Cb = (-11059 R - 21709 G + 32768 B + (128 << 16) + 32767) >> 16
 *             Cr = (32768 R - 27439 G - 5329 B + (128 << 16) + 32767) >> 16
 *   Sampling (jcsample.c), on the full-resolution Cb and Cr:
 *     444  a copy: the chroma planes are w x h.
 *     422  chroma ceil(w/2) x h; column i = (c[2i] + c[2i+1] + bias) >> 1, bias 0 at even i, 1 at odd i (h2v1_downsample).
 *     420  chroma ceil(w/2) x ceil(h/2); sample (i, j) = (the 2 x 2 box at (2i, 2j) summed + bias) >> 2, bias 1 at even i, 2 at
 *          odd i (h2v2_downsample).
 *   A ragged last column or row is replicated at full resolution before the box sums (expand_right_edge and the preprocessor's
 *   bottom-edge expansion): an odd width's last 4:2:0 sample is (2 (a + b) + bias) >> 2 of the last column's two rows.
 * Only the visible samples are written: Y is w x h, each chroma plane ceil(w / h_factor) x ceil(h / v_factor).  The caller chooses the
 * sampling (the reference lets evalchroma pick it per image).  The source is 4-byte aligned BGRA; each plane may sit at any byte
 * address with any pitch that holds a row.  4:4:0, 4:1:1, grayscale output and smoothing are not covered. */
typedef struct ifb200_bgra_to_ycbcr_desc {
    int32_t        sampling;                /* enum ifb200_ycbcr_sampling */
    const uint8_t* src; uint32_t src_stride;   /* w x h BGRA: 4-byte aligned pointer and stride; only read */
    uint8_t*       y;  uint32_t y_stride;   /* w x h luma */
    uint8_t*       cb; uint32_t cb_stride;  /* chroma planes at the sampling's size; each plane has its own pitch */
    uint8_t*       cr; uint32_t cr_stride;
    uint32_t       w, h;
    int32_t        alpha_meaningful;        /* != 0: flatten over matte_bgra first (as ifb200_batch_apply_matte) */
    uint8_t        matte_bgra[4];           /* B, G, R, A; white (255, 255, 255, 255) unless the encoder is given one */
} ifb200_bgra_to_ycbcr_desc;

/* A decoder's colour profile (the reference's SourceProfile, codecs/source_profile.rs:7-41, CMYK excluded) and the transform of a
 * frame to sRGB under it: transform_to_srgb(to_bgra(src, format), profile) as codecs/moxcms_transform.rs runs it with
 * lut_transform_opts() (relative colorimetric), for the profiles whose transform is a matrix-shaper.  Kinds:
 *   SRGB             the identity (is_srgb()): in place nothing is written; from rows the output is ifb200_batch_pixel_convert's.
 *   ICC              icc / icc_len: an ICC profile (v2 or v4) with colour space 'RGB ', PCS 'XYZ ', rXYZ / gXYZ / bXYZ and rTRC / gTRC /
 *                    bTRC tags.  A TRC is 'curv' (0 entries: identity; 1: u8Fixed8 gamma; more: a table interpolated linearly) or
 *                    'para' (function types 0-4, ICC.1:2010 §10.18; a power of a negative base is 0).
 *   ICC_GRAY         icc / icc_len: colour space 'GRAY' with a kTRC tag.  The gray value is the B byte of to_bgra(src); B, G and R all
 *                    get the transformed value, alpha is kept (moxcms_transform.rs:356-376).
 *   GAMMA_PRIMARIES  gamma: the PNG gAMA value (the encoding gamma); the TRC is x^f32(1 / gamma).  chrm: white, red, green, blue x,y.
 *   CICP             cicp = {colour primaries, transfer characteristics, matrix coefficients, full range}: primaries any code of
 *                    H.273 table 2 (1, 4-12, 22); transfer 1/6/14/15 (BT.709), 4 (gamma 2.2), 5 (gamma 2.8), 7 (SMPTE 240M),
 *                    8 (linear) or 13 (sRGB); matrix coefficients 0; full range.  Primaries 1 with transfer 13 is SRGB.
 * The plan, in float64 rounded once to f32: T_c[v] = f32(clip01(trc_c(v / 255))), v = 0..255, and M = f32(S^-1 C), where C is the
 * source colorants (rXYZ gXYZ bXYZ as stored -- chad / wtpt not applied -- or, for GAMMA_PRIMARIES and CICP, the chromaticities'
 * colorants Bradford-adapted to D50) and S the sRGB colorants (BT.709 primaries, D65) Bradford-adapted to D50 (0.9642, 1, 0.8249).
 * Per pixel, in f32 without contraction: o_c = (M[c][0] T_r[r] + M[c][1] T_g[g]) + M[c][2] T_b[b], and the byte is the resample's
 * linear-to-sRGB table at trunc(clamp(o_c * 16383, 0, 16383)) (the clamp is the clip to [0, 1], NaN -> 0).  A gray plan is one byte
 * map, gray[v] = that encode of T[v].  Alpha passes unchanged (RGB24 and Gray8 sources: 255, as to_bgra gives).
 * Refused with IFB200_ERR_NOT_IMPLEMENTED (keep such a frame on the CPU CMS): A2B0-2, B2A0-2, D2B0-3 or B2D0-3 tags; mft1, mft2,
 * 'mAB ' or 'mBA ' tag types; a Lab PCS; CMYK or any colour space but RGB and GRAY; CICP transfer PQ (16), HLG (18) or any code not
 * listed; unknown CICP primaries; matrix coefficients other than 0; narrow range.  Refused with IFB200_ERR_INVALID_ARGUMENT: a
 * truncated or malformed profile (every offset and size is checked against icc_len; nothing outside the buffer is read), a colour
 * space that does not match the kind (an RGB profile as ICC_GRAY and the reverse), a gamma or chromaticity that gives no matrix. */
enum ifb200_profile_kind { IFB200_PROFILE_SRGB = 0, IFB200_PROFILE_ICC = 1, IFB200_PROFILE_ICC_GRAY = 2,
                           IFB200_PROFILE_GAMMA_PRIMARIES = 3, IFB200_PROFILE_CICP = 4 };
typedef struct ifb200_source_profile {
    int32_t        kind;                    /* enum ifb200_profile_kind */
    const uint8_t* icc; size_t icc_len;     /* HOST bytes for the ICC kinds; read before the call returns */
    double         gamma;                   /* GAMMA_PRIMARIES: the gAMA value */
    double         chrm[8];                 /* GAMMA_PRIMARIES: white x, y, red x, y, green x, y, blue x, y */
    uint8_t        cicp[4];                 /* CICP: primaries, transfer, matrix coefficients, full range (0 / 1) */
} ifb200_source_profile;
/* What a profile plans to (ifb200_source_profile_plan). */
enum ifb200_plan_kind { IFB200_PLAN_IDENTITY = 0, IFB200_PLAN_MATRIX = 1, IFB200_PLAN_GRAY = 2 };
typedef struct ifb200_profile_plan {
    int32_t kind;                           /* enum ifb200_plan_kind */
    float   trc[3][256];                    /* MATRIX: T_r, T_g, T_b; GRAY: T in trc[0] */
    float   m[3][3];                        /* MATRIX: M[output r, g, b][input r, g, b] */
    uint8_t gray[256];                      /* GRAY: the byte map */
} ifb200_profile_plan;
/* The source of a transform: a BGRA window, or decoder rows of one of the four ifb200_pixel_op *_TO_BGRA ops. */
#define IFB200_PROFILE_SRC_BGRA 16
typedef struct ifb200_to_srgb_desc {
    int32_t        format;                  /* IFB200_PROFILE_SRC_BGRA or IFB200_PIXEL_{RGB24,RGBA,GRAY,GRAY_ALPHA}_TO_BGRA */
    const uint8_t* src; uint32_t src_stride;   /* w x h source rows; BGRA with src == dst and the same stride: in place */
    uint8_t*       dst; uint32_t dst_stride;   /* w x h BGRA destination: 4-byte aligned pointer and stride */
    uint32_t       w, h;
    const ifb200_source_profile* profile;   /* HOST pointer, read before the call returns */
} ifb200_to_srgb_desc;

/* One resample of decoder rows: scale_and_render(to_bgra(draw.in, format), canvas, params), byte for byte, without the BGRA frame
 * ever being written -- the decode -> DrawImageExact chain of a frame a GPU decoder wrote as interleaved rows (nvJPEG's RGB24, the
 * PNG and WebP decoders' RGBA32).  to_bgra is the ifb200_pixel_convert_desc op `format` with opaque = 0.
 *   draw    draw.in / in_w / in_h / in_stride: the rows as the decoder wrote them, in_w x in_h pixels; every other field as in
 *           ifb200_batch_enqueue (draw.alpha_meaningful as the caller passes it: RGB24 with alpha_meaningful = 1 resamples an alpha of 255).
 *   format  IFB200_PIXEL_RGB24_TO_BGRA (rows at any byte address, in_stride >= 3 in_w) or IFB200_PIXEL_RGBA_TO_BGRA (4-byte aligned
 *           rows and stride, in_stride >= 4 in_w).  Gray8 and GrayAlpha8 rows are refused: convert them with
 *           ifb200_batch_pixel_convert, then call ifb200_batch_enqueue. */
typedef struct ifb200_rows_resample_desc {
    ifb200_resample_desc draw;
    int32_t format;
} ifb200_rows_resample_desc;

/* One resample of oriented decoder rows: scale_and_render(orient(to_bgra(draw.in, format), orientation), canvas, params), byte for
 * byte, without the BGRA frame or the oriented frame ever being written -- a phone photo that a GPU decoder wrote as RGB24 rows, with
 * its EXIF orientation, straight into a thumbnail.
 *   draw         draw.in / in_w / in_h / in_stride: the rows as the decoder wrote them (not rotated); the resample sees in_w x in_h
 *                for 1..4 and in_h x in_w for 5..8.  Every other field as in ifb200_batch_enqueue.
 *   format       as in ifb200_rows_resample_desc, with the same row rules (checked on the stored rows).  Gray8 and GrayAlpha8 rows are
 *                refused: convert them with ifb200_batch_pixel_convert, then call ifb200_batch_enqueue_oriented.
 *   orientation  EXIF flag as in ifb200_oriented_resample_desc; values other than 2..8 are the identity.
 * The arithmetic is that of ifb200_oriented_resample_desc on the BGRA frame to_bgra gives. */
typedef struct ifb200_rows_oriented_resample_desc {
    ifb200_resample_desc draw;
    int32_t format;
    int32_t orientation;
} ifb200_rows_oriented_resample_desc;

/* One resample of a frame with a colour profile: scale_and_render(orient(transform_to_srgb(to_bgra(draw.in, format), profile),
 * orientation), canvas, params), byte for byte as ifb200_batch_transform_to_srgb followed by the matching resample entry, without the
 * sRGB frame, the BGRA frame or the oriented frame ever being written -- a Display P3 phone photo straight into a thumbnail.
 *   draw         the source as stored; every other field as in ifb200_batch_enqueue.
 *   format       IFB200_PROFILE_SRC_BGRA (a BGRA window: the rules of ifb200_batch_enqueue_oriented), or IFB200_PIXEL_RGB24_TO_BGRA /
 *                IFB200_PIXEL_RGBA_TO_BGRA (decoder rows: the rules of ifb200_batch_enqueue_rows_oriented).  Gray8 and GrayAlpha8
 *                rows are refused.
 *   orientation  EXIF flag as in ifb200_oriented_resample_desc; values other than 2..8 are the identity.
 *   profile      HOST pointer, read before the call returns; the semantics of ifb200_batch_transform_to_srgb. */
typedef struct ifb200_profiled_resample_desc {
    ifb200_resample_desc draw;
    int32_t format;
    int32_t orientation;
    const ifb200_source_profile* profile;
} ifb200_profiled_resample_desc;

/* One frame of ifb200_batch_detect_content_many: detect_content (graphics/whitespace.rs:284-331) of the DEVICE BGRA window px
 * (w x h, row pitch `stride` bytes), grayscale Bgra32 when alpha_meaningful != 0 else Bgr32, edges where the Scharr value exceeds
 * `threshold`.  The limits are those of ifb200_batch_detect_content: a non-empty window, w and h below 2^31, threshold below 2^31. */
typedef struct ifb200_detect_content_desc {
    const uint8_t* px;
    uint32_t w, h, stride;
    int32_t  alpha_meaningful;
    uint32_t threshold;
} ifb200_detect_content_desc;

/* ---- device-resident batch API (the metric path; not in the reference) -----------------------
 * descs[i].in / .canvas are DEVICE pointers on the batch's device; color_matrix stays a HOST pointer.
 * enqueue is asynchronous on `cuda_stream`, a cudaStream_t with the usual CUDA meaning (NULL = the legacy
 * default stream); pass IFB200_STREAM_OWN to use the batch's private non-blocking stream, which is the
 * stream ifb200_batch_sync waits on.  The jobs of ONE call must be independent of each other (none may read what
 * another writes): they may run concurrently.  Calls on the same stream are ordered as usual. */
#define IFB200_STREAM_OWN ((void*)(intptr_t)-1)
typedef struct ifb200_batch ifb200_batch;
int  ifb200_batch_create(int device, ifb200_batch** out, char* err, size_t err_cap);
int  ifb200_batch_enqueue(ifb200_batch* b, const ifb200_resample_desc* descs, size_t n, void* cuda_stream,
                          char* err, size_t err_cap);
/* n resamples of oriented DEVICE windows (ifb200_oriented_resample_desc), asynchronous on `cuda_stream`, as ifb200_batch_enqueue.  The
 * oriented frame is never written; the source is read as an unoriented resample reads its input.  Down-scales run the streaming ring
 * kernel, which reads its boxes through the orientation; up-scales, 1:1, windows the ring kernel cannot take (as for
 * ifb200_batch_enqueue, and with source x reversed -- flags 2, 3, 7, 8 -- a stored width that is not a multiple of four) and
 * IFB200_OPT_FORCE_GENERIC run the generic pair with an oriented H pass.  Identity jobs run exactly as ifb200_batch_enqueue runs
 * them.  Every descriptor is checked (as ifb200_batch_enqueue checks it, on the stored window) and every plan built before anything
 * is enqueued, so an error means nothing is written.  ifb200_batch_fused_jobs / ifb200_batch_generic_jobs count these jobs too. */
int  ifb200_batch_enqueue_oriented(ifb200_batch* b, const ifb200_oriented_resample_desc* d, size_t n, void* cuda_stream,
                                   char* err, size_t err_cap);
/* n resamples of DEVICE decoder rows (ifb200_rows_resample_desc), asynchronous on `cuda_stream`, as ifb200_batch_enqueue.  The BGRA
 * frame is never written: the conversion happens in the resample's source reads.  Down-scales run the streaming ring kernel (RGBA32:
 * a 16-byte aligned window and pitch, as for BGRA; RGB24: a pitch that is a multiple of 16 bytes, the window at any byte);
 * up-scales, 1:1, other windows and IFB200_OPT_FORCE_GENERIC run the generic pair with an H pass that converts its taps.  Every
 * descriptor is checked ("rows resample job i: ...") and every plan built before anything is enqueued, so an error means nothing is
 * written.  ifb200_batch_fused_jobs / ifb200_batch_generic_jobs count these jobs too. */
int  ifb200_batch_enqueue_rows(ifb200_batch* b, const ifb200_rows_resample_desc* d, size_t n, void* cuda_stream,
                               char* err, size_t err_cap);
/* n resamples of oriented DEVICE decoder rows (ifb200_rows_oriented_resample_desc), asynchronous on `cuda_stream`, as
 * ifb200_batch_enqueue.  Neither the BGRA frame nor the oriented frame is written: conversion and orientation both happen in the
 * resample's source reads.  Down-scales run the streaming ring kernel (RGBA32: the rules of ifb200_batch_enqueue_oriented; RGB24: a
 * pitch that is a multiple of 16 bytes, the window at any byte and any width); up-scales, 1:1, other windows and
 * IFB200_OPT_FORCE_GENERIC run the generic pair with an H pass that orients and converts its taps.  Identity jobs run exactly as
 * ifb200_batch_enqueue_rows runs them.  Every descriptor is checked ("oriented rows resample job i: ...") and every plan built
 * before anything is enqueued, so an error means nothing is written.  ifb200_batch_fused_jobs / ifb200_batch_generic_jobs count
 * these jobs too. */
int  ifb200_batch_enqueue_rows_oriented(ifb200_batch* b, const ifb200_rows_oriented_resample_desc* d, size_t n, void* cuda_stream,
                                        char* err, size_t err_cap);
/* n resamples of DEVICE frames with colour profiles (ifb200_profiled_resample_desc), asynchronous on `cuda_stream`, as
 * ifb200_batch_enqueue.  The transform to sRGB happens in the resample's source reads, per source pixel in the ring kernel and per tap
 * in the generic pair's H pass.  Down-scales run the streaming ring kernel under the rules of the matching entry; up-scales, 1:1,
 * other windows, forms that are not compiled (the general store epilogue: a compositing mode other than ReplaceSelf or a colour
 * matrix) and IFB200_OPT_FORCE_GENERIC run the generic pair.  Jobs whose profile plans to IFB200_PLAN_IDENTITY run exactly as
 * the matching entry runs them.  Every descriptor is checked and every distinct profile planned once before anything is enqueued,
 * so an error ("profiled resample job i: ...", with the planner's status: IFB200_ERR_NOT_IMPLEMENTED for a profile the GPU does not
 * transform -- route such frames with ifb200_source_profile_plan first) means nothing is written.  One ring launch per geometry,
 * kernel form and profile.  ifb200_batch_fused_jobs / ifb200_batch_generic_jobs count these jobs too. */
int  ifb200_batch_enqueue_profiled(ifb200_batch* b, const ifb200_profiled_resample_desc* d, size_t n, void* cuda_stream,
                                   char* err, size_t err_cap);
int  ifb200_batch_color_matrix(ifb200_batch* b, uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride,
                               const float m[25], void* cuda_stream, char* err, size_t err_cap);
int  ifb200_batch_apply_matte(ifb200_batch* b, uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride,
                              const uint8_t matte_bgra[4], int alpha_meaningful, void* cuda_stream, char* err, size_t err_cap);
int  ifb200_batch_transpose(ifb200_batch* b, const uint8_t* dev_from, uint32_t from_stride, uint32_t w, uint32_t h,
                            uint8_t* dev_to, uint32_t to_stride, void* cuda_stream, char* err, size_t err_cap);
int  ifb200_batch_flip_vertical(ifb200_batch* b, uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride,
                                void* cuda_stream, char* err, size_t err_cap);
int  ifb200_batch_flip_horizontal(ifb200_batch* b, uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride,
                                  void* cuda_stream, char* err, size_t err_cap);
int  ifb200_batch_block_scale(ifb200_batch* b, const uint8_t* dev_in, uint32_t in_stride, uint32_t blocks_x, uint32_t blocks_y,
                              uint8_t* dev_out, uint32_t out_stride, int n, int srgb, void* cuda_stream, char* err, size_t err_cap);
int  ifb200_batch_white_balance(ifb200_batch* b, uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, float threshold,
                                void* cuda_stream, char* err, size_t err_cap);
/* graphics/whitespace.rs:284-331 detect_content(&BitmapWindowMut<u8>, threshold) -> RectCorners{x1, y1, x2, y2}: the rectangle the
 * reference's whitespace scan finds (trim / `trim.threshold`).  The per-pixel arithmetic (approximate_grayscale :426-523, Scharr
 * and the local edge box :525-613) and the reference's order-dependent window walk (:333-421) both run on the GPU: this is a one-frame
 * call of ifb200_batch_detect_content_many, so the result is the reference's, not the bounding box of all edges.
 * alpha_meaningful selects the Bgra32 (1) or Bgr32 (0) grayscale.  Synchronous (a rectangle comes back). */
int  ifb200_batch_detect_content(ifb200_batch* b, const uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, int alpha_meaningful,
                                 uint32_t threshold, uint32_t rect[4], void* cuda_stream, char* err, size_t err_cap);
/* The GPU half of detect_content alone: the one-byte-per-pixel code map (layout: imageflow_b200/csrc/ifb_whitespace.h; what
 * sobel_scharr_detect :525-613 derives per 3x3 neighbourhood) of a DEVICE bitmap into a DEVICE buffer of w*h bytes, row pitch w.
 * Asynchronous on `cuda_stream`; ifb200_detect_content_from_codes() walks a host copy of it. */
int  ifb200_batch_whitespace_codes(ifb200_batch* b, const uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, int alpha_meaningful,
                                   uint32_t threshold, uint8_t* dev_codes, void* cuda_stream, char* err, size_t err_cap);
/* detect_content of n DEVICE frames (ifb200_detect_content_desc) in one call: rects[4 i .. 4 i + 3] (HOST memory) = {x1, y1, x2, y2}
 * of frame i, exactly what ifb200_batch_detect_content returns for it; visited (HOST, may be NULL) = the walk's count of
 * window-interior pixels, as ifb200_detect_content_from_codes reports it.  No code map is written: whitespace_segments_kernel reduces
 * every frame's codes into one summary per (interior row, 32-column chunk of a window column), and whitespace_walk_kernel replays the
 * reference's window order over those summaries on the device, one warp per frame (DESIGN.md §5.16).  Two kernel launches per call
 * whatever n is, none when no frame is at least 3 x 3 (those get the whole bitmap without any device work), and one device-to-host
 * copy of the results.  Every descriptor is checked before anything is launched ("detect_content job i: <why>").  Synchronous:
 * `cuda_stream` is synchronised before the call returns. */
int  ifb200_batch_detect_content_many(ifb200_batch* b, const ifb200_detect_content_desc* d, size_t n, uint32_t* rects, uint64_t* visited,
                                      void* cuda_stream, char* err, size_t err_cap);
/* Rounded corners of n DEVICE windows (d[i].px on the batch's device) in ONE kernel launch, asynchronous on `cuda_stream`.  The jobs
 * of one call must not overlap in memory (no two windows may share a pixel): they run concurrently.  Argument errors are reported
 * before anything is enqueued. */
int  ifb200_batch_round_corners(ifb200_batch* b, const ifb200_round_corners_desc* d, size_t n, void* cuda_stream, char* err, size_t err_cap);
/* Canvas operations (ifb200_canvas_desc) on n DEVICE windows in ONE kernel launch, none when no job writes a pixel; asynchronous on
 * `cuda_stream`.  No job may write what another job of the same call reads or writes; a job's input and canvas windows must not
 * overlap in memory.  Argument errors are reported before anything is enqueued.  There is no host-buffer variant: on a host bitmap
 * these ops are a memset / memcpy, cheaper than a trip to the GPU. */
int  ifb200_batch_canvas(ifb200_batch* b, const ifb200_canvas_desc* d, size_t n, void* cuda_stream, char* err, size_t err_cap);
/* Orientation (ifb200_orient_desc) of n DEVICE windows in ONE kernel launch, one read and one write per pixel whatever the flag;
 * none when no job writes a pixel (the identity in place, zero-area jobs).  Asynchronous on `cuda_stream`.  No job may write what
 * another job of the same call reads or writes (not checked).  Argument errors are reported before anything is enqueued.  There is
 * no host-buffer variant: on a host bitmap the reference's own transpose beats a trip to the GPU. */
int  ifb200_batch_orient(ifb200_batch* b, const ifb200_orient_desc* d, size_t n, void* cuda_stream, char* err, size_t err_cap);
/* Colour chains (ifb200_color_desc) of n DEVICE windows, in place: ONE kernel launch for all jobs when no job white-balances, three
 * (histograms, byte maps, apply) when any does, whatever the number of jobs; none when no job writes a pixel.  Each pixel is read
 * once and written once (read twice with a white balance).  Asynchronous on `cuda_stream`.  No two windows of a call may share a
 * pixel (not checked).  Argument errors are reported before anything is enqueued; a second WHITE_BALANCE in one job is
 * IFB200_ERR_NOT_IMPLEMENTED.  There is no host-buffer variant: on a host bitmap one pass of the reference's own loop costs less than
 * the trip to the GPU and back. */
int  ifb200_batch_color_chain(ifb200_batch* b, const ifb200_color_desc* d, size_t n, void* cuda_stream, char* err, size_t err_cap);
/* Watermarks (ifb200_watermark_desc) on n DEVICE frames, byte for byte as the node-by-node expansion (copy, Alpha, DrawImageExact).  Jobs
 * whose watermark resamples to the same premultiplied working-space image F (same source window, format, applied opacity, size, filter,
 * sharpen and working space) share ONE resample: the existing generic H pass and a V pass that stores F, one pair per distinct geometry;
 * then ONE composite launch writes every job's rectangle from its F.  Kernel launches per call: 1 + 2 x (distinct geometries), plus 1 when
 * some job has an opacity (the colour chain on the private copies); none when no job has pixels.  Device memory: the F of a call's
 * distinct watermarks (16 bytes per pixel of each) and their private copies are held at most 1 GiB at a time (plus the H pass's
 * intermediate, also at most 1 GiB, and a single F larger than that alone): a call that needs more is run as consecutive chunks of its
 * groups, each with the launches above.  Asynchronous on `cuda_stream`.  No two
 * jobs of a call may write the same pixel (not checked): several watermarks on one frame are successive calls.  A job with w or h = 0 is
 * skipped unchecked; every other descriptor is checked (as ifb200_batch_enqueue checks it, plus 4-byte aligned pointers and a NULL
 * colour matrix) and plans are built before anything is enqueued, so an error means nothing is written.  There is no host-buffer variant. */
int  ifb200_batch_watermark(ifb200_batch* b, const ifb200_watermark_desc* d, size_t n, void* cuda_stream, char* err, size_t err_cap);
/* Pixel-format conversions (ifb200_pixel_convert_desc) of n DEVICE windows in ONE kernel launch, none when no job has pixels; each
 * destination byte is written once and nothing outside the two windows is read or written.  Asynchronous on `cuda_stream`.  No job may
 * write what another job of the same call reads or writes (not checked).  Every descriptor is checked before anything is planned or
 * enqueued, so an error means nothing is written.  There is no host-buffer variant: on host rows the decoders' own loop is cheaper than
 * the trip over PCIe. */
int  ifb200_batch_pixel_convert(ifb200_batch* b, const ifb200_pixel_convert_desc* d, size_t n, void* cuda_stream, char* err, size_t err_cap);
/* JPEG colour stages (ifb200_ycbcr_desc) of n DEVICE frames in ONE kernel launch, none when no job has pixels; each destination byte is
 * written once and nothing outside the planes and the destination window is read or written.  Asynchronous on `cuda_stream`.  No job
 * may write what another job of the same call reads or writes (not checked).  Every descriptor is checked before anything is planned or
 * enqueued ("ycbcr job i: <why>", IFB200_ERR_INVALID_ARGUMENT: a null plane or destination, a stride smaller than its plane's row, an
 * unknown sampling, a misaligned destination, a destination that overlaps a plane of its job), so an error means nothing is written.
 * A job of zero area is skipped unchecked.  There is no host-buffer variant. */
int  ifb200_batch_ycbcr_to_bgra(ifb200_batch* b, const ifb200_ycbcr_desc* d, size_t n, void* cuda_stream, char* err, size_t err_cap);
/* JPEG encoder colour stages (ifb200_bgra_to_ycbcr_desc) of n DEVICE frames in ONE kernel launch, none when no job has pixels; each
 * plane byte is written once and nothing outside the source window and the planes is read or written.  Asynchronous on
 * `cuda_stream`.  No job may write what another job of the same call reads or writes (not checked).  Every descriptor is checked
 * before anything is planned or enqueued ("bgra_to_ycbcr job i: <why>", IFB200_ERR_INVALID_ARGUMENT: a null source or plane, a stride
 * smaller than its row, an unknown sampling, a misaligned source, a plane that overlaps the source or another plane of its job), so an
 * error means nothing is written.  A job of zero area is skipped unchecked.  There is no host-buffer variant. */
int  ifb200_batch_bgra_to_ycbcr(ifb200_batch* b, const ifb200_bgra_to_ycbcr_desc* d, size_t n, void* cuda_stream, char* err, size_t err_cap);
/* Colour profiles to sRGB (ifb200_to_srgb_desc, ifb200_source_profile) on n DEVICE windows in ONE kernel launch, none when no job
 * writes a pixel (SRGB jobs in place, zero-area jobs); asynchronous on `cuda_stream`.  Each destination byte is written once and
 * nothing outside the two windows is read.  Every descriptor is checked and every profile planned before anything is enqueued, so an
 * error ("transform to srgb job i: <why>", with the profile's status) means nothing is written; jobs of zero area are skipped
 * unchecked.  The row rules are ifb200_batch_pixel_convert's; overlap other than exact in-place BGRA is refused.  Identical profile
 * bytes (or parameters) within one call are planned once.  No job may write what another job of the call reads or writes (not
 * checked).  There is no host-buffer variant. */
int  ifb200_batch_transform_to_srgb(ifb200_batch* b, const ifb200_to_srgb_desc* d, size_t n, void* cuda_stream, char* err, size_t err_cap);
/* Host only, no device needed: IFB200_OK when the GPU runs this profile, IFB200_ERR_NOT_IMPLEMENTED (use the CPU CMS) or
 * IFB200_ERR_INVALID_ARGUMENT, with the reason in `why`.  When `plan` is not NULL and the status is OK, also the planned tables and
 * matrix. */
int  ifb200_source_profile_plan(const ifb200_source_profile* p, ifb200_profile_plan* plan, char* why, size_t why_cap);
int  ifb200_batch_sync(ifb200_batch* b, char* err, size_t err_cap);
void ifb200_batch_destroy(ifb200_batch* b);
/* knobs / introspection (benchmarks, tests) */
enum ifb200_option {
    IFB200_OPT_FORCE_GENERIC = 1,      /* 1: always use the two-kernel generic path (parity cross-check)  */
    IFB200_OPT_STRIP_COLUMNS = 2,      /* ring kernel: widest strip of output columns one warp works on: a multiple of 16 up to 128
                                          (default 64; clipped to what the kernel variant holds: 64, or 50 / 40 at ring depth 6) */
    IFB200_OPT_MIN_ITEMS = 3           /* ring kernel: split images into row bands until a launch has at least this many warp work
                                          items.  0 (default): as many as the device has warps, and launches that still cannot
                                          fill the device get narrower strips; > 0: exactly the strip width asked for */
};
int      ifb200_batch_set_option(ifb200_batch* b, int option, int64_t value);
uint64_t ifb200_batch_kernel_launches(const ifb200_batch* b);   /* total kernels launched so far   */
/* Where the calling thread has spent its enqueue calls so far, in seconds (inclusive: [1..4] are parts of [0]; [2] and [3] parts of [4]):
   out[0] whole enqueue calls, [1] building plans, [2] pinned staging slots (search + cudaMallocHost), [3] memcpy of tables into
   them, [4] table uploads (allocation + [2] + [3] + cudaMemcpyAsync + events); then counts: [5] table uploads, [6] bytes staged,
   [7] cudaMallocHost calls, [8] row bands of the ring kernel's launches (summed over launches).  Fills min(n, 9) entries,
   returns 9. */
int      ifb200_batch_host_profile(const ifb200_batch* b, double* out, int n);
uint64_t ifb200_batch_fused_jobs(const ifb200_batch* b);        /* jobs that took the streaming ring kernel */
uint64_t ifb200_batch_generic_jobs(const ifb200_batch* b);      /* jobs that took the generic pair */
uint64_t ifb200_batch_tile_jobs(const ifb200_batch* b);         /* jobs that took the tile kernel (up-scales, 1:1) */
/* 1 when the streaming ring kernel (the fast path for down-scales) can run on this device/driver; 0 when jobs that would take it
 * fall back to the tile kernel or the generic pair -- `why` (may be NULL) then says what is missing. */
int      ifb200_batch_ring_status(const ifb200_batch* b, char* why, size_t why_cap);

#ifdef __cplusplus
}
#endif
#endif /* IFB200_H */
