// ifb_lut.cuh -- included by ifb_kernels.cuh inside namespace ifbk (product code, sm_90a); in its own file so that tests/cpu_emu can
// include it with the kernels that use it.  Uses only __fmul_rn, fminf, fmaxf, __ldg.
// lut.rs:4-8
__device__ __forceinline__ uint32_t lut_encode(const uint8_t* __restrict__ lut16k, float lin) {
    float s = __fmul_rn(lin, 16383.0f);
    s = fminf(fmaxf(s, 0.0f), 16383.0f);     // NaN -> 0, as `NaN as usize`
    return (uint32_t)__ldg(lut16k + (int)s);
}
