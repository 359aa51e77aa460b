// ifb_pixel_convert_kernel.cuh -- included by ifb_kernels.cuh inside namespace ifbk (product code, sm_90a).  Uses only threadIdx,
// blockIdx, uint4, __byte_perm and __funnelshift_r -- tests/cpu_emu/pixel_convert_kernel_emu.cc compiles this file with g++ under a
// sequential emulation of those and checks it against tests/pixel_convert_oracle.py.
//
// The pixel-format conversions of ifb200_batch_pixel_convert: every job of a call in one flat launch over the work items of
// ifb_pixel_convert.h; each CTA finds its item by a binary search over the items' first CTAs.  Each thread owns a 16-byte group of a
// destination row, aligned to the destination's addresses: 4 BGRA pixels, or 16 bytes (5 1/3 pixels) of an RGB24 row.
//   Loads:  the source bytes of the group are fetched as the aligned 4-byte words that hold them and realigned in registers with
//           funnel shifts, so every source phase runs on word loads.  Only a word that crosses an end of the source row is read a
//           byte at a time, and then only the bytes the group needs: nothing outside the source window is read, stride padding
//           included.
//   Stores: a whole group is one 16-byte store; a group cut by an end of the row stores its whole words as words and the rest bytes.
// Each destination byte is stored once.  In place (RGBA_TO_BGRA, src == dst) every thread reads exactly the words it then writes.
#ifndef IFB_PC_LOAD1                                             // the CPU emulation defines these to record every byte accessed
#define IFB_PC_LOAD1(p) __ldcs(p)
#define IFB_PC_LOAD4(p) __ldcs(p)
#define IFB_PC_STORE1(p, v) __stcs((p), (v))
#define IFB_PC_STORE4(p, v) __stcs((p), (v))
#define IFB_PC_STORE16(p, v) __stcs((p), (v))
#endif

// Bytes [b0, b1) of the source span that starts at address v into r[0..NR) -- byte j of the span is byte j % 4 of r[j / 4], bytes
// outside [b0, b1) are 0.  [b0, b1) lies inside the source row [rs, re); v itself may lie before rs.  Words wholly inside the row are
// loaded whole, the bytes of the others one at a time.
template <int NR>
__device__ __forceinline__ void pc_fetch(uintptr_t v, int b0, int b1, uintptr_t rs, uintptr_t re, uint32_t (&r)[NR]) {
    const uint32_t o = (uint32_t)(v & 3);
    const uintptr_t a = v - o;
    uint32_t wd[NR + 1];
#pragma unroll
    for (int k = 0; k <= NR; ++k) {
        const int j0 = 4 * k - (int)o;                           // word k holds bytes [j0, j0 + 4) of the span
        const uintptr_t p = a + 4 * k;
        wd[k] = 0;
        if (j0 + 4 <= b0 || j0 >= b1) continue;
        if (p >= rs && p + 4 <= re) {
            wd[k] = IFB_PC_LOAD4(reinterpret_cast<const uint32_t*>(p));
            continue;
        }
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (j0 + i >= b0 && j0 + i < b1) wd[k] |= (uint32_t)IFB_PC_LOAD1(reinterpret_cast<const uint8_t*>(p + i)) << (8 * i);
    }
#pragma unroll
    for (int j = 0; j < NR; ++j) r[j] = __funnelshift_r(wd[j], wd[j + 1], 8 * o);
}

// byte j (a compile-time constant once unrolled) of r
template <int NR>
__device__ __forceinline__ uint32_t pc_byte(const uint32_t (&r)[NR], int j) { return (r[j >> 2] >> (8 * (j & 3))) & 0xffu; }

// BGRA -> RGB24 for a group whose byte 0 is channel M of source pixel 0 (r holds source pixels 0..5): byte q of the group is channel
// (M + q) % 3 of pixel (M + q) / 3, and channel c of an RGB pixel is byte 2 - c of its BGRA source.
template <int M>
__device__ __forceinline__ void pc_to_rgb(const uint32_t (&r)[6], uint32_t (&out)[4]) {
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        out[t] = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int q = M + 4 * t + i;
            out[t] |= pc_byte(r, 4 * (q / 3) + 2 - q % 3) << (8 * i);
        }
    }
}

// out to the 16-byte aligned group at G, bytes [q0, q1) of it only
__device__ __forceinline__ void pc_store(uintptr_t G, const uint32_t (&out)[4], uint32_t q0, uint32_t q1) {
    if (q0 == 0 && q1 == 16) {
        IFB_PC_STORE16(reinterpret_cast<uint4*>(G), make_uint4(out[0], out[1], out[2], out[3]));
        return;
    }
#pragma unroll
    for (uint32_t t = 0; t < 4; ++t) {
        const uint32_t s = 4 * t;
        if (s + 4 <= q0 || s >= q1) continue;
        if (s >= q0 && s + 4 <= q1) {
            IFB_PC_STORE4(reinterpret_cast<uint32_t*>(G + s), out[t]);
            continue;
        }
#pragma unroll
        for (uint32_t i = 0; i < 4; ++i)
            if (s + i >= q0 && s + i < q1) IFB_PC_STORE1(reinterpret_cast<uint8_t*>(G + s + i), (uint8_t)(out[t] >> (8 * i)));
    }
}

// group g of destination row y
__device__ __forceinline__ void pc_group(const ifb::PcItem& it, uint32_t y, uint32_t g) {
    const uintptr_t drow = reinterpret_cast<uintptr_t>(it.dst) + (size_t)y * it.dst_stride;
    const uintptr_t srow = reinterpret_cast<uintptr_t>(it.src) + (size_t)y * it.src_stride;
    const bool rgb_out = it.op == IFB200_PIXEL_BGRA_TO_RGB24;
    const uint32_t sb = it.op == IFB200_PIXEL_RGB24_TO_BGRA ? 3u : it.op == IFB200_PIXEL_GRAY_TO_BGRA ? 1u
                      : it.op == IFB200_PIXEL_GRAY_ALPHA_TO_BGRA ? 2u : 4u;
    const int64_t q0 = 16 * (int64_t)g - (int64_t)(drow & 15);  // the group's first byte, counted from the row's first byte
    const int64_t nbytes = (int64_t)it.w * (rgb_out ? 3 : 4);
    const int64_t lo = max(q0, (int64_t)0), hi = min(q0 + 16, nbytes);
    if (lo >= hi) return;
    const uintptr_t re = srow + (uintptr_t)it.w * sb;
    const uint32_t alpha = it.opaque ? 0xff000000u : 0u;
    uint32_t out[4];
    if (rgb_out) {
        const int64_t p0 = (q0 >= 0 ? q0 : q0 - 2) / 3;          // floor(q0 / 3): the source pixel of the group's byte 0
        const int m = (int)(q0 - 3 * p0);
        const int b0 = (int)(4 * (lo / 3 - p0)), b1 = (int)(4 * ((hi - 1) / 3 + 1 - p0));
        uint32_t r[6];
        pc_fetch(srow + 4 * p0, b0, b1, srow, re, r);
        if (m == 0) pc_to_rgb<0>(r, out);
        else if (m == 1) pc_to_rgb<1>(r, out);
        else pc_to_rgb<2>(r, out);
    } else {                                                     // 4-byte aligned rows: the group holds pixels p0 .. p0 + 3
        const int64_t p0 = q0 / 4;
        const int b0 = (int)(sb * (lo / 4 - p0)), b1 = (int)(sb * (hi / 4 - p0));
        const uintptr_t v = srow + (uintptr_t)(sb * p0);
        if (it.op == IFB200_PIXEL_RGB24_TO_BGRA) {
            uint32_t r[3];
            pc_fetch(v, b0, b1, srow, re, r);
#pragma unroll
            for (int i = 0; i < 4; ++i)
                out[i] = pc_byte(r, 3 * i + 2) | pc_byte(r, 3 * i + 1) << 8 | pc_byte(r, 3 * i) << 16 | 0xff000000u;
        } else if (it.op == IFB200_PIXEL_RGBA_TO_BGRA) {
            uint32_t r[4];
            pc_fetch(v, b0, b1, srow, re, r);
#pragma unroll
            for (int i = 0; i < 4; ++i) out[i] = __byte_perm(r[i], 0, 0x3012) | alpha;
        } else if (it.op == IFB200_PIXEL_GRAY_TO_BGRA) {
            uint32_t r[1];
            pc_fetch(v, b0, b1, srow, re, r);
#pragma unroll
            for (int i = 0; i < 4; ++i) out[i] = pc_byte(r, i) * 0x010101u | 0xff000000u;
        } else {
            uint32_t r[2];
            pc_fetch(v, b0, b1, srow, re, r);
#pragma unroll
            for (int i = 0; i < 4; ++i) out[i] = pc_byte(r, 2 * i) * 0x010101u | pc_byte(r, 2 * i + 1) << 24 | alpha;
        }
    }
    pc_store(drow + q0, out, (uint32_t)(lo - q0), (uint32_t)(hi - q0));
}

// the item i of n with first[i] <= blockIdx.x < first[i + 1] (ifb::push_first_cta's prefix)
__device__ __forceinline__ uint32_t pc_item_of(const uint32_t* __restrict__ first, uint32_t n) {
    uint32_t lo = 0, hi = n;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (first[mid] <= blockIdx.x) lo = mid;
        else hi = mid;
    }
    return lo;
}

__global__ void __launch_bounds__(256) pixel_convert_kernel(const ifb::PcItem* __restrict__ items, const uint32_t* __restrict__ first,
                                                            uint32_t n) {
    const uint32_t lo = pc_item_of(first, n);
    const ifb::PcItem it = items[lo];
    const uint64_t total = (uint64_t)it.groups * it.h, k0 = (uint64_t)(blockIdx.x - first[lo]) * ifb::kPcCtaGroups;
    if (k0 >= total) return;
    const uint32_t count = (uint32_t)min(total - k0, (uint64_t)ifb::kPcCtaGroups);
    for (uint32_t i = threadIdx.x; i < count; i += ifb::kPcThreads) {
        const uint32_t k = (uint32_t)k0 + i;
        pc_group(it, k / it.groups, k % it.groups);
    }
}
