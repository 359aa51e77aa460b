// ifb_ycbcr_enc_kernel.cuh -- included by ifb_kernels.cuh inside namespace ifbk, after ifb_pixel_convert_kernel.cuh and ifb_matte.cuh
// (product code, sm_90a).  Uses only threadIdx, blockIdx, uint4, pc_item_of and the matte helpers -- tests/cpu_emu/ycbcr_enc_kernel_emu.cc
// compiles this file with g++ under a sequential emulation of those and checks it against tests/ycbcr_enc_oracle.py.
//
// The JPEG encoder colour stage of ifb200_batch_bgra_to_ycbcr: apply_matte when alpha is meaningful, libjpeg-turbo's fixed-point
// RGB -> YCbCr (jccolor.c) and its chroma downsampling (jcsample.c: a copy at 4:4:4, h2v1 at 4:2:2, h2v2 at 4:2:0, with the last
// column and row replicated at full resolution).  Every job of a call in one flat launch over the work items of ifb_ycbcr_enc.h; each
// CTA finds its item by a binary search over the items' first CTAs.  Each thread owns a unit: the kYeRun = 8 source columns
// [8u, 8u + 8) of one row, at 4:2:0 of both rows 2j and 2j + 1 of a row pair, and writes their Y samples and the chroma samples they
// make (8 at 4:4:4, 4 at 4:2:2 and 4:2:0).  A unit starts at an even column, so every 2 x 1 or 2 x 2 box lies inside one thread, and
// the bias of chroma column 4u + i alternates with i.
//   Loads:  a row's 32 source bytes as two 16-byte loads when the run is whole and its address 16-byte aligned (a source whose rows
//           start at a 16-byte phase); otherwise, and at a row's ragged end, one 4-byte word per pixel.  Each source byte is read once
//           and nothing outside the source window is read.
//   Stores: each plane's bytes of the unit as one 8- or 4-byte store when they fill it and its address is aligned; otherwise whole
//           aligned words where they fit and single bytes around them (a plane at an odd phase, a row's ragged end).  Each plane byte
//           is stored once.
// Integer arithmetic only, apart from the matte.  The source is never written.
#ifndef IFB_YE_LOAD4                                             // the CPU emulation defines these to record every byte accessed
#define IFB_YE_LOAD4(p) __ldcs(p)
#define IFB_YE_LOAD16(p) __ldcs(p)
#define IFB_YE_STORE1(p, v) __stcs((p), (v))
#define IFB_YE_STORE4(p, v) __stcs((p), (v))
#define IFB_YE_STORE8(p, v) __stcs((p), (v))
#endif
#ifndef IFB_YE_ASSERT                                            // the CPU emulation checks that no sample needs a clamp
#define IFB_YE_ASSERT(c)
#endif

// The n (1..8) source pixels [x0, x0 + n) of source row `row`, after the matte when `alpha` (pixels past n are 0, never stored).
__device__ __forceinline__ void ye_fetch(const ifb::YeItem& it, uint32_t row, uint32_t x0, uint32_t n, const MatteLin& ml,
                                         const Tables& tb, uint32_t (&px)[ifb::kYeRun]) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(it.src) + (size_t)row * it.src_stride + 4 * (size_t)x0;
    if (n == ifb::kYeRun && (a & 15) == 0) {
        const uint4 u = IFB_YE_LOAD16(reinterpret_cast<const uint4*>(a)), v = IFB_YE_LOAD16(reinterpret_cast<const uint4*>(a + 16));
        px[0] = u.x; px[1] = u.y; px[2] = u.z; px[3] = u.w; px[4] = v.x; px[5] = v.y; px[6] = v.z; px[7] = v.w;
    } else {
#pragma unroll
        for (uint32_t k = 0; k < ifb::kYeRun; ++k) px[k] = k < n ? IFB_YE_LOAD4(reinterpret_cast<const uint32_t*>(a + 4 * k)) : 0u;
    }
    if (!it.alpha) return;
#pragma unroll
    for (uint32_t k = 0; k < ifb::kYeRun; ++k) {
        const uint32_t pa = px[k] >> 24;
        if (k >= n || pa == 255u) continue;
        px[k] = pa == 0u ? it.matte : matte_blend(px[k], pa, ml, tb);
    }
}

// jccolor.c rgb_ycc_convert of one BGRA pixel: Y, Cb, Cr
__device__ __forceinline__ void ye_ycc(uint32_t v, int& y, int& cb, int& cr) {
    const int b = (int)(v & 0xffu), g = (int)((v >> 8) & 0xffu), r = (int)((v >> 16) & 0xffu);
    y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;                                 // FIX(0.29900), FIX(0.58700), FIX(0.11400)
    cb = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;                // FIX(0.16874), FIX(0.33126), FIX(0.5)
    cr = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;                  // FIX(0.5), FIX(0.41869), FIX(0.08131)
    IFB_YE_ASSERT(y >= 0 && y <= 255 && cb >= 0 && cb <= 255 && cr >= 0 && cr <= 255);
}

// bytes 0 .. n - 1 of v to the plane bytes [a, a + n), n <= 8
__device__ __forceinline__ void ye_store(uintptr_t a, uint64_t v, uint32_t n) {
    if (n == 8 && (a & 7) == 0) {
        IFB_YE_STORE8(reinterpret_cast<unsigned long long*>(a), (unsigned long long)v);
        return;
    }
    if (n == 4 && (a & 3) == 0) {
        IFB_YE_STORE4(reinterpret_cast<uint32_t*>(a), (uint32_t)v);
        return;
    }
    for (uint32_t k = 0; k < n;) {
        const uintptr_t p = a + k;
        if ((p & 3) == 0 && k + 4 <= n) {
            IFB_YE_STORE4(reinterpret_cast<uint32_t*>(p), (uint32_t)(v >> (8 * k)));
            k += 4;
        } else {
            IFB_YE_STORE1(reinterpret_cast<uint8_t*>(p), (uint8_t)(v >> (8 * k)));
            k += 1;
        }
    }
}

__device__ __forceinline__ uintptr_t ye_at(uint8_t* plane, uint32_t stride, uint32_t row, uint32_t col) {
    return reinterpret_cast<uintptr_t>(plane) + (size_t)row * stride + col;
}

// One unit: row band `band` (row `band`, or rows 2 band and 2 band + 1 at 4:2:0), source columns [8u, 8u + n).
template <int S>
__device__ __forceinline__ void ye_unit(const ifb::YeItem& it, uint32_t band, uint32_t u, const MatteLin& ml, const Tables& tb) {
    const uint32_t x0 = ifb::kYeRun * u, n = min(ifb::kYeRun, it.w - x0);
    const uint32_t rows = S == IFB200_YCBCR_420 ? min(2u, it.h - 2 * band) : 1u, row0 = S == IFB200_YCBCR_420 ? 2 * band : band;
    int cb[ifb::kYeRun], cr[ifb::kYeRun];                       // 4:4:4 the samples; else the column sums of the unit's rows
#pragma unroll
    for (uint32_t k = 0; k < ifb::kYeRun; ++k) cb[k] = cr[k] = 0;
    for (uint32_t r = 0; r < rows; ++r) {
        uint32_t px[ifb::kYeRun];
        ye_fetch(it, row0 + r, x0, n, ml, tb, px);
        uint64_t yv = 0;
#pragma unroll
        for (uint32_t k = 0; k < ifb::kYeRun; ++k) {
            int y, b, c;
            ye_ycc(px[k], y, b, c);
            yv |= (uint64_t)y << (8 * k);
            cb[k] += b;
            cr[k] += c;
        }
        ye_store(ye_at(it.y, it.y_stride, row0 + r, x0), yv, n);
    }
    uint64_t bv = 0, rv = 0;
    uint32_t nc = n;
    if (S == IFB200_YCBCR_444) {
#pragma unroll
        for (uint32_t k = 0; k < ifb::kYeRun; ++k) {
            bv |= (uint64_t)cb[k] << (8 * k);
            rv |= (uint64_t)cr[k] << (8 * k);
        }
    } else {
        nc = (n + 1) / 2;
        // a ragged last row counts its row twice, a ragged last column its column twice (the replicated edges); at 4:2:2 the
        // "box" is the 2 x 1 pair of one row
        const int rep = S == IFB200_YCBCR_420 && rows == 1 ? 2 : 1, sh = S == IFB200_YCBCR_420 ? 2 : 1;
#pragma unroll
        for (uint32_t i = 0; i < ifb::kYeRun / 2; ++i) {
            const bool pair = 2 * i + 1 < n;
            const int bias = S == IFB200_YCBCR_420 ? 1 + (int)(i & 1) : (int)(i & 1);
            const int sb = rep * (cb[2 * i] + (pair ? cb[2 * i + 1] : cb[2 * i])), sr = rep * (cr[2 * i] + (pair ? cr[2 * i + 1] : cr[2 * i]));
            bv |= (uint64_t)((sb + bias) >> sh) << (8 * i);
            rv |= (uint64_t)((sr + bias) >> sh) << (8 * i);
        }
    }
    ye_store(ye_at(it.cb, it.cb_stride, band, x0 / (S == IFB200_YCBCR_444 ? 1 : 2)), bv, nc);
    ye_store(ye_at(it.cr, it.cr_stride, band, x0 / (S == IFB200_YCBCR_444 ? 1 : 2)), rv, nc);
}

template <int S>
__device__ __forceinline__ void ye_units(const ifb::YeItem& it, uint32_t k0, uint32_t count, const Tables& tb) {
    const MatteLin ml = it.alpha ? matte_lin(it.matte, tb) : MatteLin{0.0f, 0.0f, 0.0f, 0.0f};
    for (uint32_t t = threadIdx.x; t < count; t += ifb::kYeThreads) {
        const uint32_t k = k0 + t;
        ye_unit<S>(it, k / it.units, k % it.units, ml, tb);
    }
}

__global__ void __launch_bounds__(256) bgra_to_ycbcr_kernel(const ifb::YeItem* __restrict__ items, const uint32_t* __restrict__ first,
                                                            uint32_t n, Tables tb) {
    const uint32_t i = pc_item_of(first, n);
    const ifb::YeItem it = items[i];
    const uint64_t bands = it.sampling == IFB200_YCBCR_420 ? ((uint64_t)it.h + 1) / 2 : it.h;   // ifb::ycbcr_bands
    const uint64_t total = (uint64_t)it.units * bands;
    const uint64_t k0 = (uint64_t)(blockIdx.x - first[i]) * ifb::kYeCtaUnits;
    if (k0 >= total) return;
    const uint32_t count = (uint32_t)min(total - k0, (uint64_t)ifb::kYeCtaUnits);
    if (it.sampling == IFB200_YCBCR_420) ye_units<IFB200_YCBCR_420>(it, (uint32_t)k0, count, tb);
    else if (it.sampling == IFB200_YCBCR_422) ye_units<IFB200_YCBCR_422>(it, (uint32_t)k0, count, tb);
    else ye_units<IFB200_YCBCR_444>(it, (uint32_t)k0, count, tb);
}
