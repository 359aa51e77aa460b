// ifb_ycbcr.cc -- see ifb_ycbcr.h.  Product code: must not include or link anything from the test oracle.
#include "ifb_ycbcr.h"

#include "ifb_prepare.h"

namespace ifb {

Span span_of(const uint8_t* p, uint32_t stride, uint32_t rows, uint64_t row_bytes) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    return {a, a + (uint64_t)(rows - 1) * stride + row_bytes};
}

uint32_t ycbcr_chroma_w(int32_t sampling, uint32_t w) {
    if (sampling == IFB200_YCBCR_444) return w;
    return sampling == IFB200_YCBCR_422 || sampling == IFB200_YCBCR_420 ? (uint32_t)(((uint64_t)w + 1) / 2) : 0;
}

uint32_t ycbcr_chroma_h(int32_t sampling, uint32_t h) {
    if (sampling == IFB200_YCBCR_444 || sampling == IFB200_YCBCR_422) return h;
    return sampling == IFB200_YCBCR_420 ? (uint32_t)(((uint64_t)h + 1) / 2) : 0;
}

uint32_t ycbcr_bands(uint32_t sampling, uint32_t h) { return sampling == IFB200_YCBCR_420 ? (uint32_t)(((uint64_t)h + 1) / 2) : h; }

std::string ycbcr_check(const ifb200_ycbcr_desc& d, int* code) {
    if (code) *code = IFB200_ERR_INVALID_ARGUMENT;
    if (d.w == 0 || d.h == 0) return "";
    if (d.sampling != IFB200_YCBCR_444 && d.sampling != IFB200_YCBCR_422 && d.sampling != IFB200_YCBCR_420)
        return "unknown sampling " + std::to_string(d.sampling);
    if (!d.y) return "null Y plane pointer";
    if (!d.cb) return "null Cb plane pointer";
    if (!d.cr) return "null Cr plane pointer";
    if (!d.dst) return "null destination pointer";
    const uint32_t cw = ycbcr_chroma_w(d.sampling, d.w), ch = ycbcr_chroma_h(d.sampling, d.h);
    if (d.y_stride < d.w) return "Y stride " + std::to_string(d.y_stride) + " smaller than its plane's row of " + std::to_string(d.w) + " bytes";
    if (d.cb_stride < cw) return "Cb stride " + std::to_string(d.cb_stride) + " smaller than its plane's row of " + std::to_string(cw) + " bytes";
    if (d.cr_stride < cw) return "Cr stride " + std::to_string(d.cr_stride) + " smaller than its plane's row of " + std::to_string(cw) + " bytes";
    if (d.dst_stride < (uint64_t)d.w * 4)
        return "destination stride " + std::to_string(d.dst_stride) + " smaller than a BGRA row of " + std::to_string((uint64_t)d.w * 4) + " bytes";
    if ((reinterpret_cast<uintptr_t>(d.dst) | d.dst_stride) & 3) return "BGRA destination pointer or stride not 4-byte aligned";
    if ((uint64_t)dst_groups_per_row(d.dst, d.dst_stride, (uint64_t)d.w * 4) * ycbcr_bands(d.sampling, d.h) > 0xffffffffull)
        return "window too large";
    const Span t = span_of(d.dst, d.dst_stride, d.h, (uint64_t)d.w * 4);
    const Span planes[3] = {span_of(d.y, d.y_stride, d.h, d.w), span_of(d.cb, d.cb_stride, ch, cw), span_of(d.cr, d.cr_stride, ch, cw)};
    const char* const names[3] = {"Y", "Cb", "Cr"};
    for (int i = 0; i < 3; ++i)
        if (planes[i].a < t.b && t.a < planes[i].b) return std::string("destination overlaps the ") + names[i] + " plane";
    return "";
}

void ycbcr_plan(const ifb200_ycbcr_desc& d, YcWork& wk) {
    if (d.w == 0 || d.h == 0) return;
    YcItem it{};
    it.y = d.y; it.cb = d.cb; it.cr = d.cr; it.dst = d.dst;
    it.y_stride = d.y_stride; it.cb_stride = d.cb_stride; it.cr_stride = d.cr_stride; it.dst_stride = d.dst_stride;
    it.w = d.w; it.h = d.h; it.sampling = (uint32_t)d.sampling;
    it.groups = dst_groups_per_row(d.dst, d.dst_stride, (uint64_t)d.w * 4);
    wk.items.push_back(it);
    push_first_cta(wk.first, ((uint64_t)it.groups * ycbcr_bands(it.sampling, it.h) + kYcCtaUnits - 1) / kYcCtaUnits);
}

std::string ycbcr_prepare(const ifb200_ycbcr_desc* d, size_t n, YcWork& wk, int* code) {
    const std::string why = check_each("ycbcr", d, n, ycbcr_check, code);
    if (why.empty())
        for (size_t i = 0; i < n; ++i) ycbcr_plan(d[i], wk);
    return why;
}

}  // namespace ifb
