// ifb_orient_kernel.cuh -- included by ifb_kernels.cuh inside namespace ifbk (product code, sm_90a).  Uses only threadIdx,
// blockIdx, __syncthreads, __shared__ and uint4 -- tests/cpu_emu/orient_kernel_emu.cc compiles this file with g++ under a
// sequential emulation of those and checks it against the reference's expansion.
//
// The eight EXIF orientations of ifb200_batch_orient as one gather: one read and one write per pixel, every job of a call in one
// flat launch over the work items of ifb_orient.h.  Each CTA finds its item by a binary search over the items' first CTAs.
//   kOrTile (5..8): 32 source columns x kOrTileOx output columns through padded shared memory, as transpose_bgra8_kernel.  The
//     tile is cut in source columns and OUTPUT columns, with the reversals folded into the row indices, so that each warp reads 32
//     consecutive pixels of a source row and writes 32 consecutive pixels of an output row, both aligned to their window's first
//     column.
//   kOrRow (1..4 out of place): output rows in 16-byte groups aligned to the output's addresses; a full group whose source is
//     16-byte aligned too is one 16-byte load (its words reversed for an H-flip), every other pixel a 4-byte word.
//   kOrPair (2..4 in place): each thread swaps a group of the pair domain (ifb_orient.cc) with its mirror image.
// Every destination pixel is stored once (fixed points of an in-place flip not at all); nothing outside the windows is touched.
#ifndef IFB_OR_LOAD4                                             // the CPU emulation defines these to record every pixel access
#define IFB_OR_LOAD4(p) __ldcs(p)
#define IFB_OR_STORE4(p, v) __stcs((p), (v))
#define IFB_OR_LOAD16(p) __ldcs(p)
#define IFB_OR_STORE16(p, v) __stcs((p), (v))
#define IFB_OR_TILE(t, r, c) ((t)[r][c])
#endif

// n (1..4) consecutive pixels at p into v[0..n)
__device__ __forceinline__ void or_load(const uint32_t* p, uint32_t n, uint32_t v[4]) {
    if (n == 4 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) {
        const uint4 q = IFB_OR_LOAD16(reinterpret_cast<const uint4*>(p));
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
        return;
    }
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i)
        if (i < n) v[i] = IFB_OR_LOAD4(p + i);
}
// v[0..n) to the n pixels at p, in reverse order when rev
__device__ __forceinline__ void or_store(uint32_t* p, uint32_t n, const uint32_t v[4], bool rev) {
    if (n == 4 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) {
        IFB_OR_STORE16(reinterpret_cast<uint4*>(p), rev ? make_uint4(v[3], v[2], v[1], v[0]) : make_uint4(v[0], v[1], v[2], v[3]));
        return;
    }
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i)
        if (i < n) IFB_OR_STORE4(p + (rev ? n - 1u - i : i), v[i]);
}

// group g of row r of a kOrRow / kOrPair item
__device__ __forceinline__ void or_group(const ifb::OrItem& it, uint32_t r, uint32_t g) {
    const uint32_t y = it.y0 + r;
    uint8_t* const drow = it.out + (size_t)y * it.out_stride;
    const uint32_t a = (uint32_t)((reinterpret_cast<uintptr_t>(drow) & 15) >> 2);      // the row's first pixel is word a of its group
    const uint32_t lo = max(4 * g, a) - a, hi = min(4 * g + 4, a + it.xlim) - a;      // pixels [lo, hi) of the row
    if (lo >= hi) return;
    const uint32_t n = hi - lo;
    const bool fx = (it.flags & ifb::kOrFx) != 0, fy = (it.flags & ifb::kOrFy) != 0;
    const uint32_t sy = fy ? it.h - 1u - y : y, sx = fx ? it.w - hi : lo;             // the source of [lo, hi): [sx, sx + n)
    uint32_t* const s = const_cast<uint32_t*>(reinterpret_cast<const uint32_t*>(it.in + (size_t)sy * it.in_stride)) + sx;
    uint32_t* const d = reinterpret_cast<uint32_t*>(drow) + lo;
    uint32_t v[4] = {0, 0, 0, 0}, u[4] = {0, 0, 0, 0};
    or_load(s, n, v);
    if (it.kind == ifb::kOrPair) {                               // in place (in == out): the mirror image gets this group
        or_load(d, n, u);
        or_store(s, n, u, fx);
    }
    or_store(d, n, v, fx);
}

// CTA c of a kOrTile item: source columns [sx0, sx0 + 32) x output columns [ox0, ox0 + kOrTileOx).  Output column ox reads source
// row h-1-ox (kOrFy) or ox; source column sx lands in output row w-1-sx (kOrFx) or sx.  All loads of the CTA are issued before the
// barrier (kOrTileOx / 8 per thread), which keeps enough bytes in flight and spreads the item search over more pixels.
__device__ __forceinline__ void or_tile(const ifb::OrItem& it, uint32_t c, uint32_t (*tile)[33]) {
    const uint32_t lane = threadIdx.x & 31u, wy = threadIdx.x >> 5;
    const uint32_t sx0 = (c % it.groups) * 32u, ox0 = (c / it.groups) * ifb::kOrTileOx;
    const bool fx = (it.flags & ifb::kOrFx) != 0, fy = (it.flags & ifb::kOrFy) != 0;
#pragma unroll
    for (uint32_t j = 0; j < ifb::kOrTileOx; j += 8) {
        const uint32_t k = wy + j, ox = ox0 + k, sx = sx0 + lane;
        if (ox < it.h && sx < it.w) {
            const uint32_t sy = fy ? it.h - 1u - ox : ox;
            IFB_OR_TILE(tile, k, lane) = IFB_OR_LOAD4(reinterpret_cast<const uint32_t*>(it.in + (size_t)sy * it.in_stride) + sx);
        }
    }
    __syncthreads();
#pragma unroll
    for (uint32_t j = 0; j < 32; j += 8) {
        const uint32_t k = wy + j, sx = sx0 + k;
        if (sx >= it.w) continue;
        uint32_t* const orow = reinterpret_cast<uint32_t*>(it.out + (size_t)(fx ? it.w - 1u - sx : sx) * it.out_stride);
#pragma unroll
        for (uint32_t q = 0; q < ifb::kOrTileOx; q += 32) {
            const uint32_t ox = ox0 + q + lane;
            if (ox < it.h) IFB_OR_STORE4(orow + ox, IFB_OR_TILE(tile, q + lane, k));
        }
    }
}

__global__ void __launch_bounds__(256) orient_kernel(const ifb::OrItem* __restrict__ items, const uint32_t* __restrict__ first, uint32_t n) {
    __shared__ uint32_t tile[ifb::kOrTileOx][33];
    uint32_t lo = 0, hi = n;                                     // the item i with first[i] <= blockIdx.x < first[i + 1]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (first[mid] <= blockIdx.x) lo = mid;
        else hi = mid;
    }
    const ifb::OrItem it = items[lo];
    const uint32_t c = blockIdx.x - first[lo];
    if (it.kind == ifb::kOrTile) {
        or_tile(it, c, tile);
        return;
    }
    const uint32_t k0 = c * ifb::kOrCtaGroups;
    const uint32_t count = (uint32_t)min((uint64_t)it.groups * it.rows - k0, (uint64_t)ifb::kOrCtaGroups);
    for (uint32_t i = threadIdx.x; i < count; i += ifb::kOrThreads) {
        const uint32_t k = k0 + i;
        or_group(it, k / it.groups, k % it.groups);
    }
}
