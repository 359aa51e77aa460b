// ifb_color_kernel.cuh -- included by ifb_kernels.cuh inside namespace ifbk (product code, sm_90a).  Uses only threadIdx, blockIdx,
// __syncthreads, __shared__, uint4, atomicAdd and __ddiv_rn / __dmul_rn -- tests/cpu_emu/color_kernel_emu.cc compiles this file with
// g++ under a sequential emulation of those and checks it against the reference's node-by-node expansion.
//
// The colour chains of ifb200_batch_color_chain over the jobs of ifb_color.h.  Each CTA finds its job by a binary search over the
// jobs' first CTAs, stages the job's segments, tables and matrices in shared memory, and walks kClCtaGroups 16-byte groups of the
// job's rows (aligned to the addresses of each row; 4-byte words at ragged or misaligned ends).  Every pixel goes through all the
// job's segments in registers: a table segment is four byte gathers from shared memory, a matrix segment the reference's f32 sums
// (__fmul_rn / __fadd_rn in color_matrix.rs's order, as color_matrix_kernel).
//   color_hist_kernel   (jobs with a white balance) the segments before it, counted into per-warp shared histograms that are flushed
//                       into the job's 768 u64 counters; nothing is written to the frame.
//   color_maps_kernel   one CTA per white balance: the reference's area thresholds and byte maps into the job's kClWb table.
//   color_apply_kernel  every segment, one read and one write per pixel.
#ifndef IFB_CL_LOAD4                                             // the CPU emulation defines these to record every access
#define IFB_CL_LOAD4(p) __ldcs(p)
#define IFB_CL_STORE4(p, v) __stcs((p), (v))
#define IFB_CL_LOAD16(p) __ldcs(p)
#define IFB_CL_STORE16(p, v) __stcs((p), (v))
#define IFB_CL_SET(lhs, v) ((lhs) = (v))                         // a shared-memory store
#define IFB_CL_SHARED_ADD(p, v) atomicAdd((p), (v))
#define IFB_CL_GLOBAL_ADD(p, v) atomicAdd((p), (v))
#endif

// white_balance.rs:14-42 area_threshold over one channel's 256 counters: both scans compare against low_threshold, as the reference
// does.  Shared with white_balance_maps_kernel.
__device__ __forceinline__ void wb_area_threshold(const unsigned long long* hc, unsigned long long total_pixels, double low_threshold,
                                                  unsigned long long* lo, unsigned long long* hi) {
    const double pixel_count = (double)total_pixels;
    unsigned long long low = 0, high = 255, area = 0;
    for (int ix = 0; ix < 256; ++ix) { area += hc[ix]; if (__ddiv_rn((double)area, pixel_count) > low_threshold) { low = ix; break; } }
    area = 0;
    for (int ix = 255; ix >= 0; --ix) { area += hc[ix]; if (__ddiv_rn((double)area, pixel_count) > low_threshold) { high = ix; break; } }
    *lo = low; *hi = high;
}
// white_balance.rs:44-48 create_byte_mapping, entry v.  `high - low` is a usize subtraction in the reference: it wraps when the
// thresholds cross (release build semantics).
__device__ __forceinline__ uint8_t wb_map_byte(unsigned long long lo, unsigned long long hi, unsigned long long v) {
    const double scale = __ddiv_rn(255.0, (double)(hi - lo));
    const unsigned long long d = v > lo ? v - lo : 0ull;                                   // saturating_sub
    double m = round(__dmul_rn((double)d, scale));
    m = fmax(fmin(m, 255.0), 0.0);                                                         // NaN -> 255 -> 255, as f64::min/max
    return (uint8_t)m;
}

struct ClDev {                                                   // one launch's view of the uploaded plan
    const ifb::ClJob* jobs; const uint32_t* first; uint32_t n;
    const ifb::ClSeg* segs; uint8_t* tables; const float* mats;
    unsigned long long* hist;                                    // 768 counters per white balance (R, G, B)
};

struct ClShared {
    uint32_t tab[ifb::kClMaxSteps][256];                         // 1024-byte tables, as words
    float mat[ifb::kClMaxSteps][20];
    ifb::ClSeg seg[ifb::kClMaxSteps];
};

// the job of this CTA and the CTA's index within it
__device__ __forceinline__ uint32_t cl_find(const ClDev& a, uint32_t* c) {
    uint32_t lo = 0, hi = a.n;                                   // the job i with first[i] <= blockIdx.x < first[i + 1]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (a.first[mid] <= blockIdx.x) lo = mid;
        else hi = mid;
    }
    *c = blockIdx.x - a.first[lo];
    return lo;
}

__device__ __forceinline__ void cl_stage(const ClDev& a, const ifb::ClJob& j, ClShared& s) {
    const uint32_t* tw = reinterpret_cast<const uint32_t*>(a.tables) + (size_t)j.tab0 * 256;
    for (uint32_t i = threadIdx.x; i < j.ntab * 256; i += ifb::kClThreads) IFB_CL_SET((&s.tab[0][0])[i], tw[i]);
    for (uint32_t i = threadIdx.x; i < j.nmat * 20; i += ifb::kClThreads) IFB_CL_SET((&s.mat[0][0])[i], a.mats[(size_t)j.mat0 * 20 + i]);
    for (uint32_t i = threadIdx.x; i < j.nseg; i += ifb::kClThreads) IFB_CL_SET(s.seg[i], a.segs[j.seg0 + i]);
}

__device__ __forceinline__ uint32_t cl_lookup(const ClShared& s, uint32_t t, uint32_t byte_pos, uint32_t v) {
    const uint8_t* tb = reinterpret_cast<const uint8_t*>(s.tab[t]);
    return tb[byte_pos * 256 + v];
}

// the four pixels of a group through segments [0, nseg): each segment's matrix is read from shared memory once per group
__device__ __forceinline__ void cl_pixels(uint32_t v[4], const ClShared& s, uint32_t nseg) {
    for (uint32_t i = 0; i < nseg; ++i) {
        const ifb::ClSeg g = s.seg[i];
        if (g.kind == ifb::kClMatrix) {                          // color_matrix.rs:5-28
            float m[20];
#pragma unroll
            for (int k = 0; k < 20; ++k) m[k] = s.mat[g.idx][k];
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float fb = (float)(v[q] & 0xffu), fg = (float)((v[q] >> 8) & 0xffu), fr = (float)((v[q] >> 16) & 0xffu),
                            fa = (float)(v[q] >> 24);
                uint32_t o[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    float x = __fmul_rn(m[c * 5 + 0], fr);
                    x = __fadd_rn(x, __fmul_rn(m[c * 5 + 1], fg));
                    x = __fadd_rn(x, __fmul_rn(m[c * 5 + 2], fb));
                    x = __fadd_rn(x, __fmul_rn(m[c * 5 + 3], fa));
                    o[c] = uchar_clamp_ff(__fadd_rn(x, m[c * 5 + 4]));
                }
                v[q] = o[2] | (o[1] << 8) | (o[0] << 16) | (o[3] << 24);
            }
        } else {                                                 // kClTable / kClWb: one byte table per byte position
#pragma unroll
            for (int q = 0; q < 4; ++q)
                v[q] = cl_lookup(s, g.idx, 0, v[q] & 0xffu) | (cl_lookup(s, g.idx, 1, (v[q] >> 8) & 0xffu) << 8) |
                       (cl_lookup(s, g.idx, 2, (v[q] >> 16) & 0xffu) << 16) | (cl_lookup(s, g.idx, 3, v[q] >> 24) << 24);
        }
    }
}

// group g of row r of job j: its pixels [lo, lo + n) of the row at p (n = 0: the group is past the row's end)
__device__ __forceinline__ uint32_t* cl_group(const ifb::ClJob& j, uint32_t r, uint32_t g, uint32_t* n) {
    uint8_t* const row = j.px + (size_t)r * j.stride;
    const uint32_t a = (uint32_t)((reinterpret_cast<uintptr_t>(row) & 15) >> 2);          // the row's first pixel is word a of its group
    const uint32_t lo = max(4 * g, a) - a, hi = min(4 * g + 4, a + j.w) - a;
    *n = lo < hi ? hi - lo : 0;
    return reinterpret_cast<uint32_t*>(row) + lo;
}

__device__ __forceinline__ void cl_load(const uint32_t* p, uint32_t n, uint32_t v[4]) {
    if (n == 4 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) {
        const uint4 q = IFB_CL_LOAD16(reinterpret_cast<const uint4*>(p));
        v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
        return;
    }
#pragma unroll
    for (uint32_t i = 0; i < 4; ++i)
        if (i < n) v[i] = IFB_CL_LOAD4(p + i);
}

// the groups [k0, k0 + count) of CTA c of job j, or count = 0 past the job's end
__device__ __forceinline__ uint32_t cl_range(const ifb::ClJob& j, uint32_t c, uint32_t* k0) {
    const uint64_t total = (uint64_t)j.groups * j.h;
    *k0 = c * ifb::kClCtaGroups;
    return *k0 >= total ? 0u : (uint32_t)min(total - *k0, (uint64_t)ifb::kClCtaGroups);
}

__global__ void __launch_bounds__(256) color_apply_kernel(ClDev a) {
    __shared__ ClShared s;
    uint32_t c, k0;
    const ifb::ClJob j = a.jobs[cl_find(a, &c)];
    const uint32_t count = cl_range(j, c, &k0);
    if (count == 0) return;
    cl_stage(a, j, s);
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < count; i += ifb::kClThreads) {
        const uint32_t k = k0 + i;
        uint32_t n, v[4] = {0, 0, 0, 0};
        uint32_t* const p = cl_group(j, k / j.groups, k % j.groups, &n);
        if (n == 0) continue;
        cl_load(p, n, v);
        cl_pixels(v, s, j.nseg);
        if (n == 4 && (reinterpret_cast<uintptr_t>(p) & 15) == 0) {
            IFB_CL_STORE16(reinterpret_cast<uint4*>(p), make_uint4(v[0], v[1], v[2], v[3]));
        } else {
#pragma unroll
            for (uint32_t q = 0; q < 4; ++q)
                if (q < n) IFB_CL_STORE4(p + q, v[q]);
        }
    }
}

// jobs = the white-balancing jobs, whose nseg stops before the white balance
__global__ void __launch_bounds__(256) color_hist_kernel(ClDev a) {
    __shared__ ClShared s;
    __shared__ uint32_t hs[ifb::kClThreads / 32][768];          // one histogram per warp: R, G, B
    uint32_t c, k0;
    const ifb::ClJob j = a.jobs[cl_find(a, &c)];
    const uint32_t count = cl_range(j, c, &k0);
    if (count == 0) return;
    for (uint32_t i = threadIdx.x; i < (ifb::kClThreads / 32) * 768; i += ifb::kClThreads) IFB_CL_SET((&hs[0][0])[i], 0u);
    cl_stage(a, j, s);
    __syncthreads();
    uint32_t* const mine = hs[threadIdx.x >> 5];
    for (uint32_t i = threadIdx.x; i < count; i += ifb::kClThreads) {
        const uint32_t k = k0 + i;
        uint32_t n, v[4] = {0, 0, 0, 0};
        const uint32_t* const p = cl_group(j, k / j.groups, k % j.groups, &n);
        if (n == 0) continue;
        cl_load(p, n, v);
        cl_pixels(v, s, j.nseg);
#pragma unroll
        for (uint32_t q = 0; q < 4; ++q) {
            if (q >= n) break;
            const uint32_t x = v[q];
            IFB_CL_SHARED_ADD(&mine[(x >> 16) & 0xffu], 1u);
            IFB_CL_SHARED_ADD(&mine[256u + ((x >> 8) & 0xffu)], 1u);
            IFB_CL_SHARED_ADD(&mine[512u + (x & 0xffu)], 1u);
        }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < 768; i += ifb::kClThreads) {
        uint32_t t = 0;
#pragma unroll
        for (uint32_t w = 0; w < ifb::kClThreads / 32; ++w) t += hs[w][i];
        if (t) IFB_CL_GLOBAL_ADD(&a.hist[(size_t)j.wb * 768 + i], (unsigned long long)t);
    }
}

// one CTA of 256 threads per white balance (jobs = the white-balancing jobs): thread v writes entry v of the R, G and B maps into the
// byte positions 2, 1, 0 of the job's kClWb table.  Every thread scans the counters itself (they are the same for all threads, so
// the scans neither diverge nor need a barrier).
__global__ void __launch_bounds__(256) color_maps_kernel(ClDev a) {
    const ifb::ClJob j = a.jobs[blockIdx.x];
    const ifb::ClSeg wb = a.segs[j.seg0 + j.wb_seg];
    uint8_t* const t = a.tables + ((size_t)j.tab0 + wb.idx) * 1024;
    const unsigned long long total = (unsigned long long)j.w * j.h;
#pragma unroll 1
    for (uint32_t ch = 0; ch < 3; ++ch) {                        // R, G, B
        unsigned long long lo, hi;
        wb_area_threshold(a.hist + (size_t)j.wb * 768 + ch * 256, total, j.low, &lo, &hi);
        t[(2 - ch) * 256 + threadIdx.x] = wb_map_byte(lo, hi, threadIdx.x);
    }
}
