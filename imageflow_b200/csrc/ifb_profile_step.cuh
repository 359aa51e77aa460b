// ifb_profile_step.cuh -- the per-pixel step of a colour profile's plan (product code, sm_90a).  Included by ifb_kernels.cuh inside
// namespace ifbk, and by the kernels that run the step (ifb_profile_kernel.cuh, ifb_hv_kernel.cuh), so that tests/cpu_emu gets it with
// them.  Uses only __fmul_rn, __fadd_rn, fminf and fmaxf.
//
// One function for every kernel that applies a plan (transform_to_srgb_kernel, the ring kernel's source reads, the oriented H pass of
// the generic pair): the same operations in the same order, each kernel bringing its own table look-ups.
#pragma once

// the plan kinds (= enum ifb200_plan_kind) and the ring kernel's PROF template parameter
enum : uint32_t { PF_IDENTITY = 0u, PF_MATRIX = 1u, PF_GRAY = 2u };

// a plan as the resample kernels read it (ifb200_batch_enqueue_profiled): ifb200_profile_plan's tables without its kind, which the
// kernel form carries (the engine copies them into the launch's work upload)
struct ProfDev {
    float trc[3][256];        // MATRIX: T_r, T_g, T_b
    float m[9];               // MATRIX: M[output r, g, b][input r, g, b]
    uint8_t gray[256];        // GRAY: the byte map
};

// lut.rs:4-8 as lut_encode (ifb_lut.cuh) computes it: the index of a linear value in the 16 K linear -> sRGB table
__device__ __forceinline__ int pf_lut_index(float lin) {
    float s = __fmul_rn(lin, 16383.0f);
    s = fminf(fmaxf(s, 0.0f), 16383.0f);     // NaN -> 0, as `NaN as usize`
    return (int)s;
}

// One pixel word through a plan of kind `kind`: blue is byte BB of the word, green byte 1, red byte 2 - BB (BB = 0: BGRA; 2: the
// RGBA32 / RGB24 words of decoder rows); byte 3 (alpha) passes unchanged, and the result has the same layout.
//   GRAY    B, G, R = map[B]
//   MATRIX  o_c = (M[c][0] T_r[r] + M[c][1] T_g[g]) + M[c][2] T_b[b], no contraction, then enc(o_c)
// trc(c, v) = T_c[v] (c: 0 red, 1 green, 2 blue), gray(v) = map[v], enc(x) = the linear -> sRGB table at pf_lut_index(x).
template <uint32_t BB, class Trc, class Gray, class Enc>
__device__ __forceinline__ uint32_t pf_step(uint32_t p, uint32_t kind, const float (&m)[9], Trc&& trc, Gray&& gray, Enc&& enc) {
    constexpr uint32_t BR = 2u - BB;
    if (kind == PF_GRAY) return gray((p >> (8u * BB)) & 0xffu) * 0x010101u | (p & 0xff000000u);
    if (kind != PF_MATRIX) return p;
    const float r = trc(0, (p >> (8u * BR)) & 0xffu), g = trc(1, (p >> 8) & 0xffu), b = trc(2, (p >> (8u * BB)) & 0xffu);
    uint32_t o[3];
#pragma unroll
    for (int c = 0; c < 3; ++c)
        o[c] = enc(__fadd_rn(__fadd_rn(__fmul_rn(m[3 * c], r), __fmul_rn(m[3 * c + 1], g)), __fmul_rn(m[3 * c + 2], b)));
    return o[2] << (8u * BB) | o[1] << 8 | o[0] << (8u * BR) | (p & 0xff000000u);
}
