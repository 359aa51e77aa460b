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
 * and the local edge box :525-613) runs on the GPU for all pixels; the reference's order-dependent window walk (:333-421) is
 * replayed on the host over that one-byte-per-pixel map, so the result is the reference's, not the bounding box of all edges.
 * alpha_meaningful selects the Bgra32 (1) or Bgr32 (0) grayscale.  Synchronous (a rectangle comes back). */
int  ifb200_batch_detect_content(ifb200_batch* b, const uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, int alpha_meaningful,
                                 uint32_t threshold, uint32_t rect[4], void* cuda_stream, char* err, size_t err_cap);
/* The GPU half of detect_content alone: the one-byte-per-pixel code map (layout: imageflow_b200/csrc/ifb_whitespace.h; what
 * sobel_scharr_detect :525-613 derives per 3x3 neighbourhood) of a DEVICE bitmap into a DEVICE buffer of w*h bytes, row pitch w.
 * Asynchronous on `cuda_stream`; ifb200_detect_content_from_codes() walks a host copy of it. */
int  ifb200_batch_whitespace_codes(ifb200_batch* b, const uint8_t* dev_px, uint32_t w, uint32_t h, uint32_t stride, int alpha_meaningful,
                                   uint32_t threshold, uint8_t* dev_codes, void* cuda_stream, char* err, size_t err_cap);
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
   [7] cudaMallocHost calls.  Fills min(n, 8) entries, returns 8. */
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
