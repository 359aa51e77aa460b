// ifb_finish.cuh -- included by ifb_kernels.cuh inside namespace ifbk (product code, sm_90a); in its own file so that tests/cpu_emu can
// include the store epilogue with the kernels that use it.  Uses only __fmul_rn, __fadd_rn, __fsub_rn, __fdiv_rn, __ldg and lut_encode.
__device__ __forceinline__ uint32_t encode(bool linear, const uint8_t* __restrict__ lut16k, float v) {
    return linear ? lut_encode(lut16k, v) : uchar_clamp_ff(__fmul_rn(255.0f, v));   // color.rs:59-69
}

// Store epilogue for one destination pixel. F = premultiplied working-space (b,g,r,a).
// `dst` is read only for BlendWithSelf.  Returns packed BGRA8.
// SIMPLE = true: the caller guarantees compose == ReplaceSelf and no colour matrix (the common thumbnail case);
// the composite / matte / matrix code is then not even compiled into the kernel.
template <bool SIMPLE = false>
__device__ __forceinline__ uint32_t finish_pixel(float b, float g, float r, float a, const uint32_t flags, const JobDev& job,
                                                 const Tables& tb, const uint8_t* dst) {
    const bool linear = flags & JF_LINEAR;
    const bool am = flags & JF_ALPHA;
    const uint32_t compose = SIMPLE ? 0u : (flags >> JF_COMPOSE_SHIFT) & 3u;
    uint32_t ob, og, orr, oa;
    if (compose == 1u) {                                   // BlendWithSelf: scaling.rs:254-287
        if (a > 0.994f || !am) {
            ob = encode(linear, tb.lut16k, b); og = encode(linear, tb.lut16k, g); orr = encode(linear, tb.lut16k, r); oa = 255u;
        } else {
            const uint32_t d = *reinterpret_cast<const uint32_t*>(dst);
            const float* T = linear ? tb.t_lin : tb.t_srgb;
            const float da = (float)(int)(d >> 24);
            const float dc = __fmul_rn(__fsub_rn(1.0f, a), __fadd_rn(__fmul_rn(1.0f / 255.0f, da), 0.0f));
            const float fa = __fadd_rn(a, dc);
            ob = encode(linear, tb.lut16k, __fdiv_rn(__fadd_rn(b, __fmul_rn(dc, __ldg(T + (d & 0xffu)))), fa));
            og = encode(linear, tb.lut16k, __fdiv_rn(__fadd_rn(g, __fmul_rn(dc, __ldg(T + ((d >> 8) & 0xffu)))), fa));
            orr = encode(linear, tb.lut16k, __fdiv_rn(__fadd_rn(r, __fmul_rn(dc, __ldg(T + ((d >> 16) & 0xffu)))), fa));
            oa = uchar_clamp_ff(__fmul_rn(fa, 255.0f));
        }
    } else if (!am) {                                      // scaling.rs:227-232
        ob = encode(linear, tb.lut16k, b); og = encode(linear, tb.lut16k, g); orr = encode(linear, tb.lut16k, r); oa = 255u;
    } else {
        if (compose == 2u) {                               // BlendWithMatte (scaling.rs:119-148)
            const float t = __fsub_rn(1.0f, a);
            b = __fadd_rn(b, __fmul_rn(t, job.matte[0]));
            g = __fadd_rn(g, __fmul_rn(t, job.matte[1]));
            r = __fadd_rn(r, __fmul_rn(t, job.matte[2]));
            a = __fadd_rn(a, __fmul_rn(t, job.matte[3]));
        }
        if (a > 0.0f) { b = __fdiv_rn(b, a); g = __fdiv_rn(g, a); r = __fdiv_rn(r, a); }
        ob = encode(linear, tb.lut16k, b); og = encode(linear, tb.lut16k, g); orr = encode(linear, tb.lut16k, r);
        oa = uchar_clamp_ff(__fmul_rn(a, 255.0f));
    }
    if (!SIMPLE && (flags & JF_CM)) {                  // color_matrix.rs:5-28, on sRGB bytes
        const float fr = (float)orr, fg = (float)og, fb = (float)ob, fa = (float)oa;
        const float* m = job.cm;
        auto row = [&](int c) {
            float s = __fmul_rn(m[c * 5 + 0], fr);
            s = __fadd_rn(s, __fmul_rn(m[c * 5 + 1], fg));
            s = __fadd_rn(s, __fmul_rn(m[c * 5 + 2], fb));
            s = __fadd_rn(s, __fmul_rn(m[c * 5 + 3], fa));
            return uchar_clamp_ff(__fadd_rn(s, m[c * 5 + 4]));
        };
        orr = row(0); og = row(1); ob = row(2); oa = row(3);
    }
    return ob | (og << 8) | (orr << 16) | (oa << 24);
}
template <bool SIMPLE = false>
__device__ __forceinline__ uint32_t finish_pixel(float b, float g, float r, float a, const JobDev& job, const Tables& tb, const uint8_t* dst) {
    return finish_pixel<SIMPLE>(b, g, r, a, job.flags, job, tb, dst);
}
