// ifb_ycbcr_enc.cc -- see ifb_ycbcr_enc.h.  Product code: must not include or link anything from the test oracle.
#include "ifb_ycbcr_enc.h"

#include "ifb_prepare.h"
#include "ifb_ycbcr.h"

namespace ifb {

std::string bgra_to_ycbcr_check(const ifb200_bgra_to_ycbcr_desc& d, int* code) {
    if (code) *code = IFB200_ERR_INVALID_ARGUMENT;
    if (d.w == 0 || d.h == 0) return "";
    if (d.sampling != IFB200_YCBCR_444 && d.sampling != IFB200_YCBCR_422 && d.sampling != IFB200_YCBCR_420)
        return "unknown sampling " + std::to_string(d.sampling);
    if (!d.src) return "null source pointer";
    if (!d.y) return "null Y plane pointer";
    if (!d.cb) return "null Cb plane pointer";
    if (!d.cr) return "null Cr plane pointer";
    const uint32_t cw = ycbcr_chroma_w(d.sampling, d.w), ch = ycbcr_chroma_h(d.sampling, d.h);
    if (d.src_stride < (uint64_t)d.w * 4)
        return "source stride " + std::to_string(d.src_stride) + " smaller than a BGRA row of " + std::to_string((uint64_t)d.w * 4) + " bytes";
    if (d.y_stride < d.w) return "Y stride " + std::to_string(d.y_stride) + " smaller than its plane's row of " + std::to_string(d.w) + " bytes";
    if (d.cb_stride < cw) return "Cb stride " + std::to_string(d.cb_stride) + " smaller than its plane's row of " + std::to_string(cw) + " bytes";
    if (d.cr_stride < cw) return "Cr stride " + std::to_string(d.cr_stride) + " smaller than its plane's row of " + std::to_string(cw) + " bytes";
    if ((reinterpret_cast<uintptr_t>(d.src) | d.src_stride) & 3) return "BGRA source pointer or stride not 4-byte aligned";
    if (((uint64_t)d.w + kYeRun - 1) / kYeRun * ycbcr_bands(d.sampling, d.h) > 0xffffffffull) return "window too large";
    const Span s[4] = {span_of(d.src, d.src_stride, d.h, (uint64_t)d.w * 4), span_of(d.y, d.y_stride, d.h, d.w),
                       span_of(d.cb, d.cb_stride, ch, cw), span_of(d.cr, d.cr_stride, ch, cw)};
    const char* const names[4] = {"source", "Y plane", "Cb plane", "Cr plane"};
    for (int i = 1; i < 4; ++i)
        for (int j = 0; j < i; ++j)
            if (s[i].a < s[j].b && s[j].a < s[i].b) return std::string("the ") + names[i] + " overlaps the " + names[j];
    return "";
}

void bgra_to_ycbcr_plan(const ifb200_bgra_to_ycbcr_desc& d, YeWork& wk) {
    if (d.w == 0 || d.h == 0) return;
    YeItem it{};
    it.src = d.src; it.y = d.y; it.cb = d.cb; it.cr = d.cr;
    it.src_stride = d.src_stride; it.y_stride = d.y_stride; it.cb_stride = d.cb_stride; it.cr_stride = d.cr_stride;
    it.w = d.w; it.h = d.h; it.sampling = (uint32_t)d.sampling;
    it.units = (uint32_t)(((uint64_t)d.w + kYeRun - 1) / kYeRun);
    it.alpha = d.alpha_meaningful ? 1u : 0u;
    it.matte = (uint32_t)d.matte_bgra[0] | (uint32_t)d.matte_bgra[1] << 8 | (uint32_t)d.matte_bgra[2] << 16 | (uint32_t)d.matte_bgra[3] << 24;
    wk.items.push_back(it);
    push_first_cta(wk.first, ((uint64_t)it.units * ycbcr_bands(it.sampling, it.h) + kYeCtaUnits - 1) / kYeCtaUnits);
}

std::string bgra_to_ycbcr_prepare(const ifb200_bgra_to_ycbcr_desc* d, size_t n, YeWork& wk, int* code) {
    const std::string why = check_each("bgra_to_ycbcr", d, n, bgra_to_ycbcr_check, code);
    if (why.empty())
        for (size_t i = 0; i < n; ++i) bgra_to_ycbcr_plan(d[i], wk);
    return why;
}

}  // namespace ifb
