// ifb_kernels.cuh -- sm_90a device code of the resample hot path (product code).
//
// Stands in for the arithmetic the reference delegates to zenresize 0.3.1 behind
// graphics/scaling.rs:93-251 (resize_to_canvas / resize_with_matte / resize_and_composite),
// plus composite_premul_f32_over_srgb_u8 (scaling.rs:254-287) and
// window_bgra32_apply_color_matrix (color_matrix.rs:5-28) as store epilogues.
//
// Arithmetic contract (identical in every kernel here and in oracle/ifb_oracle.c):
//   load   p = (T[b]*af, T[g]*af, T[r]*af, af), af = a*(1/255f)     alpha meaningful   (CH = 4)
//          p = (T[b], T[g], T[r])                                    otherwise          (CH = 3)
//   H pass fmaf chain over the taps of an output column, source columns ascending, from +0   (rows are filtered as they stream in,
//   V pass fmaf chain over the H-filtered source rows of an output row, ascending, from +0    like zenresize's push_row / next_output_row)
//   store  un-premultiply (a > 0), encode, compose, optional colour matrix
// Compiled with -fmad=false: the only fused multiply-adds are the explicit __fmaf_rn below.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

#include "ifb_round_corners.h"     // RcJob / RcTile: planned on the host, read by round_corners_kernel
#include "ifb_canvas.h"            // CvItem / CvTile: planned on the host, read by canvas_kernel
#include "ifb_orient.h"            // OrItem: planned on the host, read by orient_kernel
#include "ifb_color.h"             // ClJob / ClSeg: planned on the host, read by the colour-chain kernels
#include "ifb_watermark.h"         // WmJob / WmGroup: planned on the host, read by watermark_composite_kernel
#include "ifb_pixel_convert.h"     // PcItem: planned on the host, read by pixel_convert_kernel
#include "ifb_ycbcr.h"             // YcItem: planned on the host, read by ycbcr_to_bgra_kernel
#include "ifb_ycbcr_enc.h"         // YeItem: planned on the host, read by bgra_to_ycbcr_kernel
#include "ifb_profile.h"           // PfWork: planned on the host, read by transform_to_srgb_kernel
#include "ifb_whitespace.h"        // WsSeg / WsJob / WsColumn: planned on the host, read by the detect_content_many kernels

namespace ifbk {

// ---------------------------------------------------------------- device-side descriptors (their own file: tests/cpu_emu includes it too)
#include "ifb_types.cuh"

// ---------------------------------------------------------------- scalar helpers
#include "ifb_lut.cuh"
#include "ifb_finish.cuh"
#include "ifb_profile_step.cuh"
#include "ifb_matte.cuh"

// ---------------------------------------------------------------- generic two-kernel path
// Any geometry / filter.  H pass writes a float4 intermediate [in_h][out_w]; V pass + store epilogue read it.
// Rows are folded into a loop over blockIdx.y so that no dimension of the bitmaps is bounded by a grid limit.
__global__ void __launch_bounds__(128) hpass_generic_kernel(const JobDev* __restrict__ jobs, Tables tb, AxisDev ah,
                                                            uint32_t in_h, uint32_t out_w, float4* __restrict__ inter) {
    const uint32_t X = blockIdx.x * blockDim.x + threadIdx.x;
    const JobDev& job = jobs[blockIdx.z];
    if (X >= out_w) return;
    const bool am = job.flags & JF_ALPHA;
    const float* __restrict__ T = (job.flags & JF_LINEAR) ? tb.t_lin : tb.t_srgb;
    const uint32_t l = ah.left[X], r = ah.right[X];
    const float* __restrict__ w = ah.w + ah.off[X];
    for (uint32_t j = blockIdx.y; j < in_h; j += gridDim.y) {
        const uint32_t* __restrict__ src = reinterpret_cast<const uint32_t*>(job.in + (size_t)j * job.in_stride);
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        for (uint32_t k = l; k <= r; ++k) {
            const uint32_t px = __ldg(src + k);
            const float wt = __ldg(w + (k - l));
            float pb = __ldg(T + (px & 0xffu)), pg = __ldg(T + ((px >> 8) & 0xffu)), pr = __ldg(T + ((px >> 16) & 0xffu)), pa = 0.0f;
            if (am) {
                pa = __ldg(tb.t_srgb + (px >> 24));
                pb = __fmul_rn(pb, pa); pg = __fmul_rn(pg, pa); pr = __fmul_rn(pr, pa);
            }
            a0 = __fmaf_rn(wt, pb, a0); a1 = __fmaf_rn(wt, pg, a1); a2 = __fmaf_rn(wt, pr, a2); a3 = __fmaf_rn(wt, pa, a3);
        }
        inter[((size_t)blockIdx.z * in_h + j) * out_w + X] = make_float4(a0, a1, a2, a3);
    }
}

// The H pass of the oriented resample (ifb200_batch_enqueue_oriented): the same chain, in the same order, over the taps of output
// column X of ORIENTED row j, each tap read from the stored window through the orientation (in_w x in_h is the oriented size;
// JF_FLIP_X / JF_FLIP_Y of the job).  Writes the intermediate vpass_generic_kernel reads.  TR (flags 5..8): thread = oriented row,
// blockIdx.y = output column, so that a warp's loads of one tap are consecutive pixels of one source row.
// BPP 0: BGRA frames; 3 / 4: decoder rows (ifb200_batch_enqueue_rows_oriented), each tap read and converted as hpass_rows_kernel<BPP>
// reads it (rows_tap_bgra, below).
template <int BPP>                                               // one tap of decoder rows at p as a BGRA word
__device__ __forceinline__ uint32_t rows_tap_bgra(const uint8_t* p) {
    if constexpr (BPP == 3) return (uint32_t)__ldg(p + 2) | ((uint32_t)__ldg(p + 1) << 8) | ((uint32_t)__ldg(p) << 16) | 0xff000000u;
    else return __byte_perm(__ldg(reinterpret_cast<const uint32_t*>(p)), 0u, 0x3012);
}
// PROF != PF_IDENTITY (ifb200_batch_enqueue_profiled): every tap through pf_step under the plan `prof` first, its tables read
// through __ldg (flag 1 is the form without flips).
template <bool TR, int BPP = 0, int PROF = PF_IDENTITY>
__global__ void __launch_bounds__(128) hpass_oriented_kernel(const JobDev* __restrict__ jobs, Tables tb, AxisDev ah, uint32_t in_w,
                                                             uint32_t in_h, uint32_t out_w, float4* __restrict__ inter,
                                                             const ProfDev* __restrict__ prof) {
    constexpr size_t kPx = BPP == 0 ? 4 : BPP;                   // bytes per stored pixel
    const JobDev& job = jobs[blockIdx.z];
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (TR ? in_h : out_w)) return;
    const bool am = job.flags & JF_ALPHA;
    const bool fx = job.flags & JF_FLIP_X, fy = job.flags & JF_FLIP_Y;
    const float* __restrict__ T = (job.flags & JF_LINEAR) ? tb.t_lin : tb.t_srgb;
    const uint32_t n_outer = TR ? out_w : in_h;
    for (uint32_t o = blockIdx.y; o < n_outer; o += gridDim.y) {
        const uint32_t X = TR ? o : t, j = TR ? t : o;
        // oriented (k, j) -> stored pixel: flags 1..4 (k or w-1-k, j or h-1-j), 5..8 (j or w-1-j, k or h-1-k), w x h as stored
        // (= in_w x in_h, or in_h x in_w); `line` is where oriented row j lies in the stored window, `step` the bytes between taps
        const uint32_t jj = (TR ? fx : fy) ? in_h - 1u - j : j;
        const uint8_t* line = TR ? job.in + (size_t)jj * kPx : job.in + (size_t)jj * job.in_stride;
        const size_t step = TR ? job.in_stride : kPx;
        const bool rev = TR ? fy : fx;           // the taps walk the stored axis backwards
        const uint32_t l = ah.left[X], r = ah.right[X];
        const float* __restrict__ w = ah.w + ah.off[X];
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        for (uint32_t k = l; k <= r; ++k) {
            const uint32_t ks = rev ? in_w - 1u - k : k;
            uint32_t px;                                               // the tap as a BGRA word
            if constexpr (BPP == 0) px = __ldg(reinterpret_cast<const uint32_t*>(line + (size_t)ks * step));
            else px = rows_tap_bgra<BPP>(line + (size_t)ks * step);
            if constexpr (PROF != PF_IDENTITY) {
                float m[9];
#pragma unroll
                for (int q = 0; q < 9; ++q) m[q] = PROF == PF_MATRIX ? __ldg(prof->m + q) : 0.0f;
                px = pf_step<0u>(px, (uint32_t)PROF, m, [&](int c, uint32_t v) { return __ldg(&prof->trc[c][v]); },
                                 [&](uint32_t v) { return (uint32_t)__ldg(prof->gray + v); }, [&](float x) { return lut_encode(tb.lut16k, x); });
            }
            const float wt = __ldg(w + (k - l));
            float pb = __ldg(T + (px & 0xffu)), pg = __ldg(T + ((px >> 8) & 0xffu)), pr = __ldg(T + ((px >> 16) & 0xffu)), pa = 0.0f;
            if (am) {
                pa = __ldg(tb.t_srgb + (px >> 24));
                pb = __fmul_rn(pb, pa); pg = __fmul_rn(pg, pa); pr = __fmul_rn(pr, pa);
            }
            a0 = __fmaf_rn(wt, pb, a0); a1 = __fmaf_rn(wt, pg, a1); a2 = __fmaf_rn(wt, pr, a2); a3 = __fmaf_rn(wt, pa, a3);
        }
        inter[((size_t)blockIdx.z * in_h + j) * out_w + X] = make_float4(a0, a1, a2, a3);
    }
}

// The H pass of the rows resample (ifb200_batch_enqueue_rows): hpass_generic_kernel's chain, in the same order, over the taps of
// output column X, each tap read from decoder rows of BPP bytes per pixel and converted as ifb200_pixel_convert_desc converts it
// (opaque = 0) -- RGBA32 (BPP 4): (r, g, b, a) -> (b, g, r, a), one aligned 4-byte load; RGB24 (BPP 3): (r, g, b) -> (b, g, r, 255),
// three byte loads at any address.  Writes the intermediate vpass_generic_kernel reads.
template <int BPP>
__global__ void __launch_bounds__(128) hpass_rows_kernel(const JobDev* __restrict__ jobs, Tables tb, AxisDev ah,
                                                         uint32_t in_h, uint32_t out_w, float4* __restrict__ inter) {
    const uint32_t X = blockIdx.x * blockDim.x + threadIdx.x;
    const JobDev& job = jobs[blockIdx.z];
    if (X >= out_w) return;
    const bool am = job.flags & JF_ALPHA;
    const float* __restrict__ T = (job.flags & JF_LINEAR) ? tb.t_lin : tb.t_srgb;
    const uint32_t l = ah.left[X], r = ah.right[X];
    const float* __restrict__ w = ah.w + ah.off[X];
    for (uint32_t j = blockIdx.y; j < in_h; j += gridDim.y) {
        const uint8_t* __restrict__ src = job.in + (size_t)j * job.in_stride;
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
        for (uint32_t k = l; k <= r; ++k) {
            uint32_t px;                                               // the tap as a BGRA word
            if constexpr (BPP == 3) px = rows_tap_bgra<3>(src + (size_t)k * 3);
            else px = __byte_perm(__ldg(reinterpret_cast<const uint32_t*>(src) + k), 0u, 0x3012);   // rows_tap_bgra<4>, indexed as before
            const float wt = __ldg(w + (k - l));
            float pb = __ldg(T + (px & 0xffu)), pg = __ldg(T + ((px >> 8) & 0xffu)), pr = __ldg(T + ((px >> 16) & 0xffu)), pa = 0.0f;
            if (am) {
                pa = __ldg(tb.t_srgb + (px >> 24));
                pb = __fmul_rn(pb, pa); pg = __fmul_rn(pg, pa); pr = __fmul_rn(pr, pa);
            }
            a0 = __fmaf_rn(wt, pb, a0); a1 = __fmaf_rn(wt, pg, a1); a2 = __fmaf_rn(wt, pr, a2); a3 = __fmaf_rn(wt, pa, a3);
        }
        inter[((size_t)blockIdx.z * in_h + j) * out_w + X] = make_float4(a0, a1, a2, a3);
    }
}

__global__ void __launch_bounds__(128) vpass_generic_kernel(const JobDev* __restrict__ jobs, Tables tb, AxisDev av,
                                                            uint32_t in_h, uint32_t out_w, uint32_t out_h,
                                                            const float4* __restrict__ inter) {
    const uint32_t X = blockIdx.x * blockDim.x + threadIdx.x;
    const JobDev& job = jobs[blockIdx.z];
    if (X >= out_w) return;
    const float4* __restrict__ col = inter + (size_t)blockIdx.z * in_h * out_w + X;
    for (uint32_t y = blockIdx.y; y < out_h; y += gridDim.y) {
        const uint32_t l = av.left[y], r = av.right[y];
        const float* __restrict__ w = av.w + av.off[y];
        float f0 = 0.f, f1 = 0.f, f2 = 0.f, f3 = 0.f;
        for (uint32_t j = l; j <= r; ++j) {
            const float wt = __ldg(w + (j - l));
            const float4 v = col[(size_t)j * out_w];
            f0 = __fmaf_rn(wt, v.x, f0); f1 = __fmaf_rn(wt, v.y, f1); f2 = __fmaf_rn(wt, v.z, f2); f3 = __fmaf_rn(wt, v.w, f3);
        }
        uint8_t* dst = job.out + (size_t)y * job.out_stride + (size_t)X * 4;
        *reinterpret_cast<uint32_t*>(dst) = finish_pixel(f0, f1, f2, f3, job, tb, dst);
    }
}

// ---------------------------------------------------------------- watermarks: the V pass that stores F, and the composite of every job from F; own file for tests/cpu_emu
#include "ifb_watermark_kernel.cuh"

// ---------------------------------------------------------------- tile kernel (up-scales, 1:1, mild down-scales; its own file: tests/cpu_emu runs this source on the CPU)
#ifndef IFB_DYNAMIC_SMEM                                 // (tests/cpu_emu defines it as a pointer to an exactly-sized heap block)
#define IFB_DYNAMIC_SMEM(name_) extern __shared__ __align__(16) unsigned char name_[]
#endif
#include "ifb_tile2_kernel.cuh"

// ---------------------------------------------------------------- standalone colour matrix (color_matrix.rs:5-28)
__global__ void __launch_bounds__(256) color_matrix_kernel(uint8_t* __restrict__ px, uint32_t w, uint32_t h, uint32_t stride,
                                                           const float* __restrict__ m20) {
    __shared__ float m[20];
    if (threadIdx.x < 20) m[threadIdx.x] = m20[threadIdx.x];
    __syncthreads();
    // The thread's pixels are counted before the loop: on a frame of more than 2^32 - step pixels (the host bounds w * h to
    // 2^32 - 1), `i < total` after a wrapping `i += step` would hold again and start another pass over finished pixels.
    const uint32_t total = w * h, step = gridDim.x * blockDim.x, first = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n = first < total ? (total - 1u - first) / step + 1u : 0u;
    uint32_t i = first;
    for (uint32_t k = 0; k < n; ++k, i += step) {
        const uint32_t y = i / w, x = i - y * w;
        uint32_t* p = reinterpret_cast<uint32_t*>(px + (size_t)y * stride) + x;
        const uint32_t v = *p;
        const float fb = (float)(v & 0xffu), fg = (float)((v >> 8) & 0xffu), fr = (float)((v >> 16) & 0xffu), fa = (float)(v >> 24);
        uint32_t o[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float s = __fmul_rn(m[c * 5 + 0], fr);
            s = __fadd_rn(s, __fmul_rn(m[c * 5 + 1], fg));
            s = __fadd_rn(s, __fmul_rn(m[c * 5 + 2], fb));
            s = __fadd_rn(s, __fmul_rn(m[c * 5 + 3], fa));
            o[c] = uchar_clamp_ff(__fadd_rn(s, m[c * 5 + 4]));
        }
        *p = o[2] | (o[1] << 8) | (o[0] << 16) | (o[3] << 24);
    }
}

// ---------------------------------------------------------------- apply_matte (graphics/blend.rs:6-59)
// Encoder-side flatten over a solid colour, in place, linear light (SURVEY.md section 8(f), item 2).
__global__ void __launch_bounds__(256) apply_matte_kernel(uint8_t* __restrict__ px, uint32_t w, uint32_t h, uint32_t stride,
                                                          uint32_t matte_bgra, Tables tb) {
    const MatteLin ml = matte_lin(matte_bgra, tb);
    const uint32_t total = w * h, step = gridDim.x * blockDim.x, first = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t n = first < total ? (total - 1u - first) / step + 1u : 0u;     // counted first, as in color_matrix_kernel
    uint32_t i = first;
    for (uint32_t k = 0; k < n; ++k, i += step) {
        const uint32_t y = i / w, x = i - y * w;
        uint32_t* p = reinterpret_cast<uint32_t*>(px + (size_t)y * stride) + x;
        const uint32_t v = *p;
        const uint32_t pa = v >> 24;
        if (pa == 0u) { *p = matte_bgra; continue; }
        if (pa == 255u) continue;
        *p = matte_blend(v, pa, ml, tb);
    }
}

// ---------------------------------------------------------------- transpose / flips (SURVEY.md section 8(f), item 3)
// Pure data movement on BGRA8 words, bound by HBM: 4 bytes read + 4 bytes written per pixel.
// graphics/transpose.rs:95-121 (bitmap_window_transpose): to[x][y] = from[y][x].  32x32-word tiles through shared memory
// (padded to 33 columns: conflict-free), 32x8 threads, both the reads and the writes are full 128-byte rows.
__global__ void __launch_bounds__(256) transpose_bgra8_kernel(const uint8_t* __restrict__ from, uint32_t from_stride, uint32_t w, uint32_t h,
                                                              uint8_t* __restrict__ to, uint32_t to_stride) {
    __shared__ uint32_t tile[32][33];
    const uint32_t x0 = blockIdx.x * 32u, y0 = blockIdx.y * 32u;
#pragma unroll
    for (int j = 0; j < 32; j += 8) {
        const uint32_t x = x0 + threadIdx.x, y = y0 + threadIdx.y + j;
        if (x < w && y < h) tile[threadIdx.y + j][threadIdx.x] = __ldcs(reinterpret_cast<const uint32_t*>(from + (size_t)y * from_stride) + x);
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < 32; j += 8) {
        const uint32_t oy = x0 + threadIdx.y + j, ox = y0 + threadIdx.x;      // destination row = source column
        if (oy < w && ox < h) __stcs(reinterpret_cast<uint32_t*>(to + (size_t)oy * to_stride) + ox, tile[threadIdx.x][threadIdx.y + j]);
    }
}
// graphics/flip.rs:10-22 (flow_bitmap_bgra_flip_vertical_safe): rows y and h-1-y swap, in place; the middle row of an odd
// height stays.  One thread per element of the top half; T = uint4 (four pixels) when rows are 16-byte aligned and the
// width is a multiple of 4, else uint32_t.
template <class T>
__global__ void __launch_bounds__(256) flip_vertical_bgra8_kernel(uint8_t* __restrict__ px, uint32_t w_elems, uint32_t h, uint32_t stride) {
    const uint32_t half = h / 2u;
    const uint64_t total = (uint64_t)half * w_elems;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t y = (uint32_t)(i / w_elems), x = (uint32_t)(i - (uint64_t)y * w_elems);
        T* a = reinterpret_cast<T*>(px + (size_t)y * stride) + x;
        T* b = reinterpret_cast<T*>(px + (size_t)(h - 1u - y) * stride) + x;
        const T va = *a, vb = *b;
        *a = vb; *b = va;
    }
}
// graphics/flip.rs:25-39 (flow_bitmap_bgra_flip_horizontal_safe): every row reversed pixel-wise, in place.
__global__ void __launch_bounds__(256) flip_horizontal_bgra8_kernel(uint8_t* __restrict__ px, uint32_t w, uint32_t h, uint32_t stride) {
    const uint32_t half = w / 2u;
    const uint64_t total = (uint64_t)half * h;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t y = (uint32_t)(i / half), x = (uint32_t)(i - (uint64_t)y * half);
        uint32_t* row = reinterpret_cast<uint32_t*>(px + (size_t)y * stride);
        const uint32_t va = row[x], vb = row[w - 1u - x];
        row[x] = vb; row[w - 1u - x] = va;
    }
}
// the same on groups of four pixels (rows 16-byte aligned, width a multiple of 4): group g swaps with group n-1-g, each
// reversed inside; the middle group of an odd count is reversed in place
__global__ void __launch_bounds__(256) flip_horizontal_bgra8_v4_kernel(uint8_t* __restrict__ px, uint32_t w4, uint32_t h, uint32_t stride) {
    const uint32_t per_row = (w4 + 1u) / 2u;
    const uint64_t total = (uint64_t)per_row * h;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t y = (uint32_t)(i / per_row), g = (uint32_t)(i - (uint64_t)y * per_row);
        uint4* row = reinterpret_cast<uint4*>(px + (size_t)y * stride);
        const uint4 a = row[g], b = row[w4 - 1u - g];
        row[g] = make_uint4(b.w, b.z, b.y, b.x);
        row[w4 - 1u - g] = make_uint4(a.w, a.z, a.y, a.x);      // g == w4-1-g (middle group): both stores write the same value
    }
}

// ---------------------------------------------------------------- colour chains (ColorMatrixSrgb, EnableTransparency, white balance) in one pass; own file for tests/cpu_emu
#include "ifb_color_kernel.cuh"

// ---------------------------------------------------------------- white balance (SURVEY.md section 8(f), item 4, first half)
// flow/nodes/white_balance.rs:93-121 = three passes: per-channel histograms (graphics/histogram.rs:7-20), the area-threshold
// byte mappings (white_balance.rs:14-48, f64 arithmetic, a handful of operations), and the in-place remap (:50-67).
// hist[0..255] = R, [256..511] = G, [512..767] = B (histogram.rs: "histogram order is RGB").
// One private histogram per warp (8 x 768 counters = 24 KB of shared memory): lanes of a warp still collide on popular bins,
// warps do not.  V4: rows are 16-byte aligned and the width is a multiple of 4 -> four pixels per load.
template <bool V4>
__global__ void __launch_bounds__(256) histogram_bgra8_kernel(const uint8_t* __restrict__ px, uint32_t w, uint32_t h, uint32_t stride,
                                                              unsigned long long* __restrict__ hist) {
    __shared__ uint32_t sh[8][768];
    for (int i = threadIdx.x; i < 8 * 768; i += 256) (&sh[0][0])[i] = 0u;
    __syncthreads();
    uint32_t* mine = sh[threadIdx.x >> 5];
    auto count = [&](uint32_t v) {
        atomicAdd(&mine[(v >> 16) & 0xffu], 1u);
        atomicAdd(&mine[256u + ((v >> 8) & 0xffu)], 1u);
        atomicAdd(&mine[512u + (v & 0xffu)], 1u);
    };
    const uint32_t we = V4 ? w / 4u : w;
    const uint64_t total = (uint64_t)we * h;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t y = (uint32_t)(i / we), x = (uint32_t)(i - (uint64_t)y * we);
        if (V4) {
            const uint4 v = __ldcs(reinterpret_cast<const uint4*>(px + (size_t)y * stride) + x);
            count(v.x); count(v.y); count(v.z); count(v.w);
        } else {
            count(__ldcs(reinterpret_cast<const uint32_t*>(px + (size_t)y * stride) + x));
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 768; i += 256) {
        uint32_t c = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) c += sh[k][i];
        if (c) atomicAdd(&hist[i], (unsigned long long)c);
    }
}
// white_balance.rs:14-48.  One block of 256 threads: thread c < 3 scans channel c's histogram from both ends (both scans
// compare against low_threshold, as the reference does), then thread v writes maps[c * 256 + v] for the three channels.
// `high - low` is a usize subtraction in the reference: it wraps when the thresholds cross (release build semantics).
// The arithmetic is wb_area_threshold / wb_map_byte (ifb_color_kernel.cuh), shared with the colour chain's color_maps_kernel.
__global__ void __launch_bounds__(256) white_balance_maps_kernel(const unsigned long long* __restrict__ hist, unsigned long long total_pixels,
                                                                 double low_threshold, uint8_t* __restrict__ maps) {
    __shared__ unsigned long long lo[3], hi[3];
    const int t = threadIdx.x;
    if (t < 3) {
        unsigned long long l, h;
        wb_area_threshold(hist + t * 256, total_pixels, low_threshold, &l, &h);
        lo[t] = l; hi[t] = h;
    }
    __syncthreads();
#pragma unroll
    for (int c = 0; c < 3; ++c) maps[c * 256 + t] = wb_map_byte(lo[c], hi[c], (unsigned long long)t);
}
// white_balance.rs:50-67: r, g, b through their byte maps, alpha untouched, in place
template <bool V4>
__global__ void __launch_bounds__(256) apply_byte_maps_bgra8_kernel(uint8_t* __restrict__ px, uint32_t w, uint32_t h, uint32_t stride,
                                                                    const uint8_t* __restrict__ maps) {
    __shared__ uint8_t sm[768];
    for (int i = threadIdx.x; i < 768; i += 256) sm[i] = maps[i];
    __syncthreads();
    auto remap = [&](uint32_t v) {
        return (v & 0xff000000u) | ((uint32_t)sm[(v >> 16) & 0xffu] << 16) | ((uint32_t)sm[256u + ((v >> 8) & 0xffu)] << 8) | (uint32_t)sm[512u + (v & 0xffu)];
    };
    const uint32_t we = V4 ? w / 4u : w;
    const uint64_t total = (uint64_t)we * h;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t y = (uint32_t)(i / we), x = (uint32_t)(i - (uint64_t)y * we);
        if (V4) {
            uint4* p = reinterpret_cast<uint4*>(px + (size_t)y * stride) + x;
            const uint4 v = *p;
            *p = make_uint4(remap(v.x), remap(v.y), remap(v.z), remap(v.w));
        } else {
            uint32_t* p = reinterpret_cast<uint32_t*>(px + (size_t)y * stride) + x;
            *p = remap(*p);
        }
    }
}

// ---------------------------------------------------------------- whitespace detection (SURVEY.md section 8(f), item 4, second half)
// In its own file so that tests/ can also execute this very source under a CPU emulation of the CUDA built-ins it uses.
#include "ifb_whitespace_kernel.cuh"

// ---------------------------------------------------------------- rounded corners (SURVEY.md section 8(f), item 5); own file for tests/cpu_emu
#include "ifb_round_corners_kernel.cuh"

// ---------------------------------------------------------------- canvas operations (fill, copy, expand, normalise alpha); own file for tests/cpu_emu
#include "ifb_canvas_kernel.cuh"

// ---------------------------------------------------------------- orientation (ApplyOrientation, rotations, flips, transpose) as one gather; own file for tests/cpu_emu
#include "ifb_orient_kernel.cuh"

// ---------------------------------------------------------------- pixel formats at the graph's edges (RGB24, RGBA, Gray, GrayAlpha <-> BGRA); own file for tests/cpu_emu
#include "ifb_pixel_convert_kernel.cuh"
#include "ifb_ycbcr_kernel.cuh"
#include "ifb_ycbcr_enc_kernel.cuh"

// ---------------------------------------------------------------- colour profiles to sRGB (matrix-shaper ICC, gray ICC, gAMA+cHRM, CICP); own file for tests/cpu_emu
#include "ifb_profile_kernel.cuh"

// ---------------------------------------------------------------- decode-time JPEG block scalers (SURVEY.md section 8(f), item 1)
#include "ifb_idct_kernel.cuh"

// ---------------------------------------------------------------- the hot kernel: streaming H-then-V ring kernel (TMA-staged rows)
#include "ifb_hv_kernel.cuh"

}  // namespace ifbk
