// ifb_profile_kernel.cuh -- included by ifb_kernels.cuh inside namespace ifbk, after ifb_lut.cuh and ifb_pixel_convert_kernel.cuh
// (product code, sm_90a).  Uses only threadIdx, blockIdx, __shared__, __syncthreads, __fmul_rn / __fadd_rn and what those two files
// use -- tests/cpu_emu/transform_to_srgb_kernel_emu.cc compiles this file with g++ under a sequential emulation of those and checks it
// against tests/profile_oracle.py.
//
// ifb200_batch_transform_to_srgb: every job of a call in one flat launch over pixel_convert's work items (ifb_profile.h), each CTA
// finding its item by a binary search over the items' first CTAs.  A CTA stages its job's plan -- three 256-entry f32 tone tables and
// the 3 x 3 matrix, or the gray byte map -- in shared memory; the 16 KB linear-to-sRGB table is read through __ldg by lut_encode (it
// stays in L1).  Each thread owns a 16-byte group of 4 destination pixels, aligned to the destination's addresses, and reads its source
// bytes with pixel_convert's pc_fetch (aligned words realigned in registers; bytes only at a row's ragged ends, nothing outside the
// source window) and writes with pc_store.  Each destination byte is stored once; in place every thread reads exactly the words it
// then writes.
//   matrix  o_c = (M[c][0] T_r[r] + M[c][1] T_g[g]) + M[c][2] T_b[b], no contraction, then lut_encode
//   gray    B, G, R = map[B]
// Alpha passes unchanged (255 from RGB24 and Gray8 rows, as to_bgra gives).

#include "ifb_profile_step.cuh"
static_assert(PF_IDENTITY == (uint32_t)IFB200_PLAN_IDENTITY && PF_MATRIX == (uint32_t)IFB200_PLAN_MATRIX && PF_GRAY == (uint32_t)IFB200_PLAN_GRAY, "plan kinds");

struct PfShared {
    float trc[3][256];
    uint8_t gray[256];
};

// one BGRA pixel through the plan (pf_step)
__device__ __forceinline__ uint32_t pf_pixel(uint32_t p, const PfShared& s, uint32_t kind, const float (&m)[9],
                                             const uint8_t* __restrict__ lut16k) {
    return pf_step<0u>(p, kind, m, [&](int c, uint32_t v) { return s.trc[c][v]; }, [&](uint32_t v) { return (uint32_t)s.gray[v]; },
                       [&](float x) { return lut_encode(lut16k, x); });
}

// group g of destination row y: to_bgra of the source as pixel_convert_kernel computes it (opaque = 0; a BGRA source as it is), then
// every pixel through the plan
__device__ __forceinline__ void pf_group(const ifb::PcItem& it, bool bgra, const PfShared& s, uint32_t kind, const float (&m)[9],
                                         const uint8_t* __restrict__ lut16k, uint32_t y, uint32_t g) {
    const uintptr_t drow = reinterpret_cast<uintptr_t>(it.dst) + (size_t)y * it.dst_stride;
    const uintptr_t srow = reinterpret_cast<uintptr_t>(it.src) + (size_t)y * it.src_stride;
    const uint32_t sb = it.op == IFB200_PIXEL_RGB24_TO_BGRA ? 3u : it.op == IFB200_PIXEL_GRAY_TO_BGRA ? 1u
                      : it.op == IFB200_PIXEL_GRAY_ALPHA_TO_BGRA ? 2u : 4u;
    const int64_t q0 = 16 * (int64_t)g - (int64_t)(drow & 15);  // the group's first byte, counted from the row's first byte
    const int64_t lo = max(q0, (int64_t)0), hi = min(q0 + 16, (int64_t)it.w * 4);
    if (lo >= hi) return;
    const uintptr_t re = srow + (uintptr_t)it.w * sb;
    const int64_t p0 = q0 / 4;                                   // 4-byte aligned rows: the group holds pixels p0 .. p0 + 3
    const int b0 = (int)(sb * (lo / 4 - p0)), b1 = (int)(sb * (hi / 4 - p0));
    const uintptr_t v = srow + (uintptr_t)(sb * p0);
    uint32_t out[4];
    if (it.op == IFB200_PIXEL_RGB24_TO_BGRA) {
        uint32_t r[3];
        pc_fetch(v, b0, b1, srow, re, r);
#pragma unroll
        for (int i = 0; i < 4; ++i) out[i] = pc_byte(r, 3 * i + 2) | pc_byte(r, 3 * i + 1) << 8 | pc_byte(r, 3 * i) << 16 | 0xff000000u;
    } else if (it.op == IFB200_PIXEL_RGBA_TO_BGRA) {
        uint32_t r[4];
        pc_fetch(v, b0, b1, srow, re, r);
#pragma unroll
        for (int i = 0; i < 4; ++i) out[i] = bgra ? r[i] : __byte_perm(r[i], 0, 0x3012);
    } else if (it.op == IFB200_PIXEL_GRAY_TO_BGRA) {
        uint32_t r[1];
        pc_fetch(v, b0, b1, srow, re, r);
#pragma unroll
        for (int i = 0; i < 4; ++i) out[i] = pc_byte(r, i) * 0x010101u | 0xff000000u;
    } else {
        uint32_t r[2];
        pc_fetch(v, b0, b1, srow, re, r);
#pragma unroll
        for (int i = 0; i < 4; ++i) out[i] = pc_byte(r, 2 * i) * 0x010101u | pc_byte(r, 2 * i + 1) << 24;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) out[i] = pf_pixel(out[i], s, kind, m, lut16k);
    pc_store(drow + q0, out, (uint32_t)(lo - q0), (uint32_t)(hi - q0));
}

// plan_of[i]: the plan of items[i] | ifb::kPfBgra for a BGRA source
__global__ void __launch_bounds__(256) transform_to_srgb_kernel(const ifb::PcItem* __restrict__ items, const uint32_t* __restrict__ first,
                                                                const uint32_t* __restrict__ plan_of,
                                                                const ifb200_profile_plan* __restrict__ plans,
                                                                const uint8_t* __restrict__ lut16k, uint32_t n) {
    __shared__ PfShared s;
    uint32_t lo = 0, hi = n;                                     // the item i with first[i] <= blockIdx.x < first[i + 1]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (first[mid] <= blockIdx.x) lo = mid;
        else hi = mid;
    }
    const ifb::PcItem it = items[lo];
    const uint64_t total = (uint64_t)it.groups * it.h, k0 = (uint64_t)(blockIdx.x - first[lo]) * ifb::kPcCtaGroups;
    if (k0 >= total) return;
    const uint32_t pj = plan_of[lo];
    const ifb200_profile_plan& pl = plans[pj & ~ifb::kPfBgra];
    const uint32_t kind = (uint32_t)pl.kind;
    if (kind == IFB200_PLAN_MATRIX)
        for (uint32_t i = threadIdx.x; i < 3 * 256; i += ifb::kPcThreads) (&s.trc[0][0])[i] = (&pl.trc[0][0])[i];
    else if (kind == IFB200_PLAN_GRAY)
        for (uint32_t i = threadIdx.x; i < 256; i += ifb::kPcThreads) s.gray[i] = pl.gray[i];
    __syncthreads();
    float m[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) m[k] = (&pl.m[0][0])[k];
    const uint32_t count = (uint32_t)min(total - k0, (uint64_t)ifb::kPcCtaGroups);
    for (uint32_t i = threadIdx.x; i < count; i += ifb::kPcThreads) {
        const uint32_t k = (uint32_t)k0 + i;
        pf_group(it, (pj & ifb::kPfBgra) != 0, s, kind, m, lut16k, k / it.groups, k % it.groups);
    }
}
