// ifb_watermark_kernel.cuh -- included by ifb_kernels.cuh inside namespace ifbk, after the store epilogue (ifb_finish.cuh) and the
// generic pair (product code, sm_90a).  Uses only threadIdx, blockIdx, blockDim, gridDim, float4, uint4, __fmaf_rn and what
// finish_pixel uses -- tests/cpu_emu/watermark_kernel_emu.cc compiles this file with g++ under a sequential emulation of those.
//
// ifb200_batch_watermark: F = the resampled premultiplied working-space watermark (float4 [h][w]) depends only on the watermark and
// the draw's geometry, filter and working space, so N frames that get the same watermark share one F, and each frame costs one
// composite = finish_pixel(F, dst) with its own compose flags -- the store epilogue of every resample kernel, byte for byte.
#ifndef IFB_WM_LOAD4                                             // the CPU emulation defines these to record every pixel access
#define IFB_WM_LOAD4(p) (*(p))
#define IFB_WM_STORE4(p, v) (*(p) = (v))
#define IFB_WM_LOAD16(p) (*(p))
#define IFB_WM_STORE16(p, v) (*(p) = (v))
#define IFB_WM_LOADF(p) (*(p))
#endif

// The V pass of the generic pair (vpass_generic_kernel: the same fmaf chain, source rows ascending from +0) storing F instead of calling
// finish_pixel.  blockIdx.z = the group among those of one geometry; their intermediates and F are consecutive.
__global__ void __launch_bounds__(128) vpass_f_kernel(AxisDev av, uint32_t in_h, uint32_t out_w, uint32_t out_h,
                                                      const float4* __restrict__ inter, float4* __restrict__ f) {
    const uint32_t X = blockIdx.x * blockDim.x + threadIdx.x;
    if (X >= out_w) return;
    const float4* __restrict__ col = inter + (size_t)blockIdx.z * in_h * out_w + X;
    float4* __restrict__ fz = f + (size_t)blockIdx.z * out_h * out_w + X;
    for (uint32_t y = blockIdx.y; y < out_h; y += gridDim.y) {
        const uint32_t l = av.left[y], r = av.right[y];
        const float* __restrict__ w = av.w + av.off[y];
        float f0 = 0.f, f1 = 0.f, f2 = 0.f, f3 = 0.f;
        for (uint32_t j = l; j <= r; ++j) {
            const float wt = __ldg(w + (j - l));
            const float4 v = col[(size_t)j * out_w];
            f0 = __fmaf_rn(wt, v.x, f0); f1 = __fmaf_rn(wt, v.y, f1); f2 = __fmaf_rn(wt, v.z, f2); f3 = __fmaf_rn(wt, v.w, f3);
        }
        fz[(size_t)y * out_w] = make_float4(f0, f1, f2, f3);
    }
}

// One launch over the jobs of groups[0, n_groups): every job of a call, or of one chunk of its groups (ifb_engine.cu watermark_locked);
// blockIdx.x is CTA cta0 + blockIdx.x of the call's numbering.  Each CTA finds its group by a binary search over the groups' first
// CTAs; inside a group the CTAs run tile by tile and, inside a tile, job by job (consecutive CTAs read the same F rows).  A thread takes a 16-byte group of a
// canvas row (aligned to the canvas' addresses, as canvas_kernel): a full group is one 16-byte load (BlendWithSelf only) and one 16-byte
// store, every other pixel a 4-byte word.  Only F and the job's rectangle are read; only the rectangle is written, each pixel once.
__global__ void __launch_bounds__(256) watermark_composite_kernel(const ifb::WmGroup* __restrict__ groups, uint32_t n_groups,
                                                                  const ifb::WmJob* __restrict__ jobs, Tables tb, uint32_t cta0) {
    const uint32_t cta = cta0 + blockIdx.x;
    uint32_t lo = 0, hi = n_groups;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (groups[mid].first <= cta) lo = mid;
        else hi = mid;
    }
    const ifb::WmGroup g = groups[lo];
    const uint32_t c = cta - g.first, tile = c / g.n;
    const ifb::WmJob job = jobs[g.job0 + (c - tile * g.n)];
    JobDev jd;                                    // finish_pixel reads the matte only (flags never carry JF_CM)
    jd.matte[0] = job.matte[0]; jd.matte[1] = job.matte[1]; jd.matte[2] = job.matte[2]; jd.matte[3] = job.matte[3];
    const uint32_t flags = job.flags & (JF_LINEAR | JF_ALPHA | (3u << JF_COMPOSE_SHIFT));
    const bool self = ((flags >> JF_COMPOSE_SHIFT) & 3u) == 1u;
    const uint32_t y0 = tile * g.rows, rows = min(g.rows, g.h - y0);
    const float4* __restrict__ F = reinterpret_cast<const float4*>(g.f);
    for (uint32_t k = threadIdx.x; k < rows * job.groups; k += ifb::kWmThreads) {
        const uint32_t r = k / job.groups, q = k - r * job.groups, y = y0 + r;
        uint8_t* const drow = job.out + (size_t)y * job.stride;
        const uint32_t a = (uint32_t)((reinterpret_cast<uintptr_t>(drow) & 15) >> 2);      // the row's first pixel is word a of its group
        const uint32_t x0 = max(4 * q, a) - a, x1 = min(4 * q + 4, a + g.w) - a;          // pixels [x0, x1) of the row
        if (x0 >= x1) continue;
        uint32_t* const d = reinterpret_cast<uint32_t*>(drow) + x0;
        const float4* const fr = F + (size_t)y * g.w + x0;
        if (x1 - x0 == 4) {
            uint4 v = make_uint4(0u, 0u, 0u, 0u);
            if (self) v = IFB_WM_LOAD16(reinterpret_cast<const uint4*>(d));
            const uint32_t in[4] = {v.x, v.y, v.z, v.w};
            uint32_t o[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const float4 p = IFB_WM_LOADF(fr + i);
                o[i] = finish_pixel(p.x, p.y, p.z, p.w, flags, jd, tb, reinterpret_cast<const uint8_t*>(in + i));
            }
            IFB_WM_STORE16(reinterpret_cast<uint4*>(d), make_uint4(o[0], o[1], o[2], o[3]));
        } else {
            for (uint32_t i = 0; i < x1 - x0; ++i) {
                const uint32_t in = self ? IFB_WM_LOAD4(d + i) : 0u;
                const float4 p = IFB_WM_LOADF(fr + i);
                IFB_WM_STORE4(d + i, finish_pixel(p.x, p.y, p.z, p.w, flags, jd, tb, reinterpret_cast<const uint8_t*>(&in)));
            }
        }
    }
}
