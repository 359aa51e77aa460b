// ifb_orient.cc -- see ifb_orient.h.  Product code: must not include or link anything from the test oracle.
#include "ifb_orient.h"

#include <algorithm>

#include "ifb_prepare.h"

namespace ifb {
namespace {

std::string check_window(const char* what, const uint8_t* p, uint32_t w, uint32_t h, uint32_t stride) {
    if (!p) return std::string("null ") + what + " pointer";
    if (reinterpret_cast<uintptr_t>(p) & 3) return std::string(what) + " pointer not 4-byte aligned";
    if (stride < w * 4ull || (stride & 3)) return std::string(what) + " stride smaller than a BGRA row or not a multiple of 4";
    return "";
}

// bytes [first, end) that a non-empty window spans
void span(const uint8_t* p, uint32_t w, uint32_t h, uint32_t stride, uintptr_t* first, uintptr_t* end) {
    *first = reinterpret_cast<uintptr_t>(p);
    *end = *first + (uint64_t)(h - 1) * stride + (uint64_t)w * 4;
}

bool transposing(int32_t o) { return o >= 5; }

void add(OrWork& wk, const OrItem& it, uint64_t ctas) {
    if (ctas == 0) return;
    if (wk.first.empty()) wk.first.push_back(0);
    wk.items.push_back(it);
    wk.first.push_back((uint32_t)std::min<uint64_t>(wk.first.back() + ctas, 0xffffffffull));
}

void add_groups(OrWork& wk, OrItem it, uint32_t y0, uint32_t rows, uint32_t xlim) {
    if (rows == 0 || xlim == 0) return;
    it.y0 = y0; it.rows = rows; it.xlim = xlim;
    it.groups = groups_per_row(it.out + (size_t)y0 * it.out_stride, it.out_stride, xlim);
    add(wk, it, ((uint64_t)it.groups * rows + kOrCtaGroups - 1) / kOrCtaGroups);
}

}  // namespace

// With a stride that is a multiple of 16 every row starts at the phase of row0; otherwise a row may start at any of the four, and
// (xlim + 6) / 4 covers the widest case.
uint32_t groups_per_row(const uint8_t* row0, uint32_t stride, uint32_t xlim) {
    const uint32_t a0 = (uint32_t)((reinterpret_cast<uintptr_t>(row0) & 15) >> 2);
    return (stride & 15) == 0 ? (a0 + xlim + 3) / 4 : (xlim + 6) / 4;
}

int32_t orient_flag(int32_t o) { return o >= 2 && o <= 8 ? o : 1; }

std::string orient_check(const ifb200_orient_desc& d, int* code) {
    if (code) *code = IFB200_ERR_INVALID_ARGUMENT;
    if (d.in_w == 0 || d.in_h == 0) return "";
    if ((uint64_t)d.in_w * d.in_h > 0xffffffffull) return "window too large";
    const int32_t o = orient_flag(d.orientation);
    const uint32_t ow = transposing(o) ? d.in_h : d.in_w, oh = transposing(o) ? d.in_w : d.in_h;
    std::string e = check_window("input", d.in, d.in_w, d.in_h, d.in_stride);
    if (e.empty()) e = check_window("output", d.out, ow, oh, d.out_stride);
    if (!e.empty()) return e;
    if (d.out == d.in) {
        if (transposing(o)) return "orientation " + std::to_string(o) + " transposes and cannot run in place";
        if (d.out_stride != d.in_stride) return "in place with a different output stride";
        return "";
    }
    uintptr_t a0, a1, b0, b1;
    span(d.in, d.in_w, d.in_h, d.in_stride, &a0, &a1);
    span(d.out, ow, oh, d.out_stride, &b0, &b1);
    if (a0 < b1 && b0 < a1) return "input and output windows overlap without being the same window";
    return "";
}

void orient_plan(const ifb200_orient_desc& d, OrWork& wk) {
    const uint32_t w = d.in_w, h = d.in_h;
    if (w == 0 || h == 0) return;
    const int32_t o = orient_flag(d.orientation);
    OrItem it{};
    it.in = d.in; it.out = d.out; it.in_stride = d.in_stride; it.out_stride = d.out_stride; it.w = w; it.h = h;
    if (transposing(o)) {                          // 5 (y, x)  6 (y, h-1-x)  7 (w-1-y, h-1-x)  8 (w-1-y, x)
        it.kind = kOrTile;
        it.flags = (o == 7 || o == 8 ? kOrFx : 0) | (o == 6 || o == 7 ? kOrFy : 0);
        it.groups = (w + 31) / 32;
        add(wk, it, (uint64_t)it.groups * ((h + kOrTileOx - 1) / kOrTileOx));
        return;
    }
    it.flags = (o == 2 || o == 3 ? kOrFx : 0) | (o == 3 || o == 4 ? kOrFy : 0);
    if (d.out != d.in) {
        it.kind = kOrRow;
        add_groups(wk, it, 0, h, w);
        return;
    }
    // in place: every pixel p with p < σ(p) once, fixed points not at all
    it.kind = kOrPair;
    if (o == 2) {
        add_groups(wk, it, 0, h, w / 2);           // the middle column of an odd width stays
    } else if (o == 4) {
        add_groups(wk, it, 0, h / 2, w);           // the middle row of an odd height stays
    } else if (o == 3) {
        add_groups(wk, it, 0, h / 2, w);
        if (h & 1) add_groups(wk, it, h / 2, 1, w / 2);   // the middle row swaps within itself; its middle pixel stays
    }
}

std::string orient_prepare(const ifb200_orient_desc* d, size_t n, OrWork& wk, int* code) {
    const std::string why = check_each("orient", d, n, orient_check, code);
    if (why.empty())
        for (size_t i = 0; i < n; ++i) orient_plan(d[i], wk);
    return why;
}

}  // namespace ifb
