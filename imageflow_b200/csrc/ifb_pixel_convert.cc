// ifb_pixel_convert.cc -- see ifb_pixel_convert.h.  Product code: must not include or link anything from the test oracle.
#include "ifb_pixel_convert.h"

#include <algorithm>

#include "ifb_prepare.h"

namespace ifb {
namespace {

const char* op_name(int32_t op) {
    static const char* const names[] = {"RGB24_TO_BGRA", "RGBA_TO_BGRA", "GRAY_TO_BGRA", "GRAY_ALPHA_TO_BGRA", "BGRA_TO_RGB24"};
    return names[op];
}

}  // namespace

// The rows' phases modulo 16 are row0's plus multiples of gcd(stride, 16), so the latest any row starts in its first group is
// (row0 mod g) + 16 - g.
uint32_t dst_groups_per_row(const uint8_t* row0, uint32_t stride, uint64_t bytes) {
    uint32_t g = 16;
    while (stride % g) g >>= 1;
    const uint32_t late = (uint32_t)(reinterpret_cast<uintptr_t>(row0) % g) + 16 - g;
    return (uint32_t)std::min<uint64_t>((late + bytes + 15) / 16, 0xffffffffull);
}

void push_first_cta(std::vector<uint32_t>& first, uint64_t ctas) {
    if (first.empty()) first.push_back(0);
    first.push_back((uint32_t)std::min<uint64_t>(first.back() + ctas, 0xffffffffull));
}

uint32_t pixel_src_bytes(int32_t op) {
    switch (op) {
        case IFB200_PIXEL_RGB24_TO_BGRA: return 3;
        case IFB200_PIXEL_RGBA_TO_BGRA: case IFB200_PIXEL_BGRA_TO_RGB24: return 4;
        case IFB200_PIXEL_GRAY_TO_BGRA: return 1;
        case IFB200_PIXEL_GRAY_ALPHA_TO_BGRA: return 2;
        default: return 0;
    }
}

uint32_t pixel_dst_bytes(int32_t op) {
    if (op == IFB200_PIXEL_BGRA_TO_RGB24) return 3;
    return pixel_src_bytes(op) ? 4 : 0;
}

std::string pixel_convert_check(const ifb200_pixel_convert_desc& d, int* code) {
    if (code) *code = IFB200_ERR_INVALID_ARGUMENT;
    if (d.w == 0 || d.h == 0) return "";
    const uint32_t sb = pixel_src_bytes(d.op), db = pixel_dst_bytes(d.op);
    if (!sb) return "unknown op " + std::to_string(d.op);
    if (!d.src) return "null source pointer";
    if (!d.dst) return "null destination pointer";
    if (d.src_stride < (uint64_t)d.w * sb) return std::string("source stride smaller than a row of ") + op_name(d.op);
    if (d.dst_stride < (uint64_t)d.w * db) return std::string("destination stride smaller than a row of ") + op_name(d.op);
    if (db == 4 && ((reinterpret_cast<uintptr_t>(d.dst) | d.dst_stride) & 3))
        return "BGRA destination pointer or stride not 4-byte aligned";
    if ((uint64_t)dst_groups_per_row(d.dst, d.dst_stride, (uint64_t)d.w * db) * d.h > 0xffffffffull) return "window too large";
    if (d.src == d.dst) {
        if (d.op != IFB200_PIXEL_RGBA_TO_BGRA) return std::string(op_name(d.op)) + " cannot run in place";
        if (d.src_stride != d.dst_stride) return "in place with a different destination stride";
        return "";
    }
    const uintptr_t a0 = reinterpret_cast<uintptr_t>(d.src), a1 = a0 + (uint64_t)(d.h - 1) * d.src_stride + (uint64_t)d.w * sb;
    const uintptr_t b0 = reinterpret_cast<uintptr_t>(d.dst), b1 = b0 + (uint64_t)(d.h - 1) * d.dst_stride + (uint64_t)d.w * db;
    if (a0 < b1 && b0 < a1) return "source and destination overlap without being the same window";
    return "";
}

void pixel_convert_plan(const ifb200_pixel_convert_desc& d, PcWork& wk) {
    if (d.w == 0 || d.h == 0) return;
    PcItem it{};
    it.src = d.src; it.dst = d.dst; it.src_stride = d.src_stride; it.dst_stride = d.dst_stride; it.w = d.w; it.h = d.h;
    it.op = (uint32_t)d.op; it.opaque = d.opaque ? 1u : 0u;
    it.groups = dst_groups_per_row(d.dst, d.dst_stride, (uint64_t)d.w * pixel_dst_bytes(d.op));
    wk.items.push_back(it);
    push_first_cta(wk.first, ((uint64_t)it.groups * it.h + kPcCtaGroups - 1) / kPcCtaGroups);
}

std::string pixel_convert_prepare(const ifb200_pixel_convert_desc* d, size_t n, PcWork& wk, int* code) {
    const std::string why = check_each("pixel convert", d, n, pixel_convert_check, code);
    if (why.empty())
        for (size_t i = 0; i < n; ++i) pixel_convert_plan(d[i], wk);
    return why;
}

}  // namespace ifb
