// ifb_round_corners_kernel.cuh -- included by ifb_kernels.cuh inside namespace ifbk, after ifb_types.cuh and ifb_lut.cuh (product
// code, sm_90a).  Uses only: threadIdx, blockIdx, __ldg, __fadd_rn, __fsub_rn, __fmul_rn, __fdiv_rn, __fsqrt_rn, __uint2float_rn,
// fabsf, floorf, ceilf, fminf, fmaxf -- tests/cpu_emu/round_corners_kernel_emu.cc compiles this file with g++ under a sequential
// emulation of those and checks it against the CPU oracle.
//
// flow_bitmap_bgra_clear_around_rounded_corners (graphics/rounded_corners.rs:187-346), one thread per pixel of the planned cover
// (ifb_round_corners.h).  The reference walks its steps one after another -- the circle-mode top fill, then per quadrant (TopLeft,
// TopRight, BottomLeft, BottomRight) the circle-mode bottom fill, the edge clears and the arc rows -- and the quadrants' rows and
// columns overlap when radii are mixed or fractional, so a later step can read what an earlier one wrote.  Every step either leaves
// a pixel alone, overwrites it with the matte, or blends the matte over the pixel's own current value: so each thread replays all
// steps in that order on its one pixel, in a register, and the result is the sequential one.  A pixel is read only if a step
// blends it (and no earlier step filled it) and written only if a step fills or blends it.
#ifndef IFB_RC_LOAD                                              // the CPU emulation defines these to record every pixel access
#define IFB_RC_LOAD(p) (*(p))
#define IFB_RC_STORE(p, v) (*(p) = (v))
#endif
__device__ __forceinline__ uint64_t rc_usize(float f) {          // `f32 as usize`: saturating, NaN -> 0
    if (!(f > 0.0f)) return 0ull;
    if (f >= 18446744073709551616.0f) return ~0ull;
    return (uint64_t)f;
}

__device__ __forceinline__ void rc_pixel(const ifb::RcJob& J, uint32_t x, uint32_t y, const Tables& tb) {
    uint32_t* const p = reinterpret_cast<uint32_t*>(J.px + (size_t)y * J.stride) + x;
    uint32_t v = 0;
    bool have = false, dirty = false;                            // v holds the pixel's current value / a step wrote it
    auto fill = [&] { v = J.matte; have = dirty = true; };
    if (y < J.top_rows) fill();                                  // :209-212
    const float a2f = 1.0f / 255.0f;
#pragma unroll 1
    for (int qi = 0; qi < 4; ++qi) {
        const ifb::RcQuad& q = J.q[qi];
        if (qi == 2 && y >= J.bottom_from) fill();               // :213-216, in the BottomLeft step
        if (y >= q.start_y && y < q.end_y) {                     // :264-343
            const float yf = __fadd_rn(__uint2float_rn(y), 0.5f);
            const float ydist = fabsf(__fsub_rn(q.cy, yf));
            const float yd2 = __fmul_rn(ydist, ydist);
            const float xds = __fsqrt_rn(fmaxf(__fsub_rn(q.ros2, yd2), 0.0f));
            const float xdi = __fsqrt_rn(fmaxf(__fsub_rn(q.roi2, yd2), 0.0f));
            bool alias = false;
            if (q.is_left) {
                const uint64_t influence_x1 = rc_usize(fmaxf(floorf(__fsub_rn(q.cx, xdi)), 0.0f));
                const uint64_t solid_x1 = rc_usize(fmaxf(ceilf(__fsub_rn(q.cx, xds)), 0.0f));
                if (x < influence_x1) { fill(); continue; }
                alias = x < solid_x1;
            } else {
                const float wf = __uint2float_rn(J.w);
                const uint64_t solid_x2 = rc_usize(fminf(floorf(__fadd_rn(q.cx, xds)), wf));
                const uint64_t influence_x2 = rc_usize(fminf(ceilf(__fadd_rn(q.cx, xdi)), wf));
                if (x >= influence_x2) { fill(); continue; }
                alias = x >= solid_x2;
            }
            if (!alias) continue;
            const float dx = __fsub_rn(q.cx, __fadd_rn(__uint2float_rn(x), 0.5f));
            const float distance = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), yd2));
            if (distance > q.roi) { fill(); continue; }
            if (!(distance > q.ros)) continue;
            const float intensity = __fdiv_rn(__fsub_rn(distance, q.ros), q.raw);
            if (!have) { v = IFB_RC_LOAD(p); have = true; }
            const float pa = __fmul_rn(__fmul_rn(__uint2float_rn(v >> 24), a2f), __fsub_rn(1.0f, intensity));
            const float ma = __fmul_rn(__fsub_rn(1.0f, pa), __fmul_rn(__uint2float_rn(J.matte >> 24), a2f));
            const float fa = __fadd_rn(ma, pa);
            auto ch = [&](int s) {
                const float lin = __fdiv_rn(__fadd_rn(__fmul_rn(__ldg(tb.t_lin + ((v >> s) & 0xffu)), pa),
                                                      __fmul_rn(__ldg(tb.t_lin + ((J.matte >> s) & 0xffu)), ma)), fa);
                return lut_encode(tb.lut16k, lin);               // final_a == 0 (both transparent): NaN -> LUT entry 0, as the reference
            };
            const uint32_t nb = ch(0), ng = ch(8), nr = ch(16);
            v = nb | (ng << 8) | (nr << 16) | (uchar_clamp_ff(__fmul_rn(255.0f, fa)) << 24);
            dirty = true;
        } else if (q.clear_from != q.clear_to && y >= q.y && y < q.bottom && x >= q.clear_from && x < q.clear_to) {
            fill();                                              // :242-250, rows of the quadrant outside its arc rows
        }
    }
    if (dirty) IFB_RC_STORE(p, v);
}

__global__ void __launch_bounds__(256) round_corners_kernel(const ifb::RcJob* __restrict__ jobs, const ifb::RcTile* __restrict__ tiles, Tables tb) {
    const ifb::RcTile t = tiles[blockIdx.x];
    const ifb::RcJob& J = jobs[t.job];
    for (uint32_t i = threadIdx.x; i < t.count; i += ifb::kRcThreads) {
        const uint32_t k = t.first + i;
        rc_pixel(J, t.x0 + k % t.rw, t.y0 + k / t.rw, tb);
    }
}
