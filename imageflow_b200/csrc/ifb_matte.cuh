// ifb_matte.cuh -- included by ifb_kernels.cuh inside namespace ifbk (product code, sm_90a); in its own file so that tests/cpu_emu
// can include it with the kernels that use it.  Uses only __fmul_rn, __fadd_rn, __fsub_rn, __fdiv_rn, __ldg, lut_encode and
// uchar_clamp_ff.
//
// Bitmap::apply_matte (graphics/blend.rs:6-59) per pixel, the encoder-side flatten over a solid colour in linear light: a pixel of
// alpha 0 becomes the matte, one of alpha 255 is kept, any other is blended.  apply_matte_kernel (in place) and
// bgra_to_ycbcr_kernel (into a JPEG encoder's planes) both run it, so their flattened pixels are the same bytes.

// the matte's alpha / 255 and its B, G, R in linear light
struct MatteLin { float a, b, g, r; };

__device__ __forceinline__ MatteLin matte_lin(uint32_t matte_bgra, const Tables& tb) {
    const float a2f = 1.0f / 255.0f;
    return {__fmul_rn((float)(matte_bgra >> 24), a2f), __ldg(tb.t_lin + (matte_bgra & 0xffu)),
            __ldg(tb.t_lin + ((matte_bgra >> 8) & 0xffu)), __ldg(tb.t_lin + ((matte_bgra >> 16) & 0xffu))};
}

// the flattened BGRA word of pixel v, whose alpha pa = v >> 24 is neither 0 nor 255
__device__ __forceinline__ uint32_t matte_blend(uint32_t v, uint32_t pa, const MatteLin& m, const Tables& tb) {
    const float a2f = 1.0f / 255.0f;
    const float paf = __fmul_rn((float)(int)pa, a2f);
    const float m_a = __fmul_rn(__fsub_rn(1.0f, paf), m.a);
    const float fa = __fadd_rn(m_a, paf);
    auto ch = [&](uint32_t byte, float mc) {
        const float lin = __fdiv_rn(__fadd_rn(__fmul_rn(__ldg(tb.t_lin + byte), paf), __fmul_rn(mc, m_a)), fa);
        return lut_encode(tb.lut16k, lin);
    };
    const uint32_t nb = ch(v & 0xffu, m.b), ng = ch((v >> 8) & 0xffu, m.g), nr = ch((v >> 16) & 0xffu, m.r);
    return nb | (ng << 8) | (nr << 16) | (uchar_clamp_ff(__fmul_rn(255.0f, fa)) << 24);
}
