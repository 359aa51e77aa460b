// ifb_canvas.cc -- see ifb_canvas.h.  Product code: must not include or link anything from the test oracle.
#include "ifb_canvas.h"

#include <algorithm>
#include <cstdio>

#include "ifb_prepare.h"

namespace ifb {
namespace {

struct Rect { uint32_t x, y, w, h; };

std::string fmt(const char* f, unsigned long long a = 0, unsigned long long b = 0, unsigned long long c = 0, unsigned long long d = 0) {
    char s[256];
    snprintf(s, sizeof s, f, a, b, c, d);
    return s;
}

std::string check_window(const char* what, const uint8_t* p, uint32_t w, uint32_t h, uint32_t stride) {
    if (!p) return std::string("null ") + what + " pointer";
    if (reinterpret_cast<uintptr_t>(p) & 3) return std::string(what) + " pointer not 4-byte aligned";
    if (stride < w * 4ull || (stride & 3)) return std::string(what) + " stride smaller than a BGRA row or not a multiple of 4";
    if ((uint64_t)w * h > 0xffffffffull) return std::string(what) + " window too large";
    return "";
}

// bytes [first, end) that a window spans (empty for an empty window)
void span(const uint8_t* p, uint32_t w, uint32_t h, uint32_t stride, uintptr_t* first, uintptr_t* end) {
    *first = reinterpret_cast<uintptr_t>(p);
    *end = (w == 0 || h == 0) ? *first : *first + (uint64_t)(h - 1) * stride + (uint64_t)w * 4;
}
bool overlap(const ifb200_canvas_desc& d) {
    uintptr_t a0, a1, b0, b1;
    span(d.px, d.w, d.h, d.stride, &a0, &a1);
    span(d.in, d.in_w, d.in_h, d.in_stride, &b0, &b1);
    return a0 < a1 && b0 < b1 && a0 < b1 && b0 < a1;
}

// The pixels of a W x H window outside the rectangle r (which lies inside it), as up to four disjoint rectangles: the rows above
// and below r across the whole width, and the parts of r's rows left and right of it.
void outside(uint32_t W, uint32_t H, const Rect& r, std::vector<Rect>& out) {
    if (r.y > 0) out.push_back({0, 0, W, r.y});
    if (r.y + r.h < H) out.push_back({0, r.y + r.h, W, H - r.y - r.h});
    if (r.x > 0) out.push_back({0, r.y, r.x, r.h});
    if (r.x + r.w < W) out.push_back({r.x + r.w, r.y, W - r.x - r.w, r.h});
}

uint32_t pack(const uint8_t c[4]) { return (uint32_t)c[0] | ((uint32_t)c[1] << 8) | ((uint32_t)c[2] << 16) | ((uint32_t)c[3] << 24); }

void add(CvWork& wk, CvKind kind, uint32_t flags, uint32_t color, uint8_t* base, uint32_t stride, const Rect& r,
         uint8_t* src_base = nullptr, uint32_t src_stride = 0, uint32_t sx = 0, uint32_t sy = 0) {
    if (r.w == 0 || r.h == 0) return;
    CvItem it{};
    it.dst = base + (size_t)r.y * stride + (size_t)r.x * 4;
    it.src = src_base ? src_base + (size_t)sy * src_stride + (size_t)sx * 4 : nullptr;
    it.dst_stride = stride; it.src_stride = src_stride; it.w = r.w; it.h = r.h;
    it.kind = kind; it.flags = flags; it.color = color;
    // A row that starts at word a (0..3) of a 16-byte group spans (a + w + 3) / 4 groups.  With a stride that is a multiple of 16
    // every row starts at the same word; otherwise a row may start at any of them, and (w + 6) / 4 covers the widest case.
    const uint32_t a0 = (uint32_t)((reinterpret_cast<uintptr_t>(it.dst) & 15) >> 2);
    it.groups = (stride & 15) == 0 ? (a0 + r.w + 3) / 4 : (r.w + 6) / 4;
    const uint32_t i = (uint32_t)wk.items.size();
    wk.items.push_back(it);
    const uint64_t area = (uint64_t)it.groups * r.h;
    for (uint64_t f = 0; f < area; f += kCvTileGroups)
        wk.tiles.push_back({i, (uint32_t)f, (uint32_t)std::min<uint64_t>(kCvTileGroups, area - f)});
}

// copy_rectangle (copy_rect.rs:47-97) of the validated rectangle (fx, fy) -> (tx, ty), cw x ch, from a window of format in_am into
// a canvas of format am
void plan_copy(const ifb200_canvas_desc& d, bool am, bool in_am, uint32_t fx, uint32_t fy, uint32_t tx, uint32_t ty, uint32_t cw, uint32_t ch,
               CvWork& wk) {
    std::vector<Rect> rest;
    uint32_t flags = 0;
    if (!am && in_am) {                              // :47-54: the canvas is normalised, then the copy overwrites the rectangle
        outside(d.w, d.h, {tx, ty, cw, ch}, rest);
        for (const Rect& r : rest) add(wk, kCvOpaque, 0, 0, d.px, d.stride, r);
    } else if (am && !in_am) {                       // :64-66: the whole input is normalised in place; the copied part by the copy
        outside(d.in_w, d.in_h, {fx, fy, cw, ch}, rest);
        for (const Rect& r : rest) add(wk, kCvOpaque, 0, 0, d.in, d.in_stride, r);
        flags = kCvOrAlpha | kCvWriteBack;
    }
    add(wk, kCvCopy, flags, 0, d.px, d.stride, {tx, ty, cw, ch}, d.in, d.in_stride, fx, fy);
}

}  // namespace

std::string canvas_check(const ifb200_canvas_desc& d, int* code) {
    if (code) *code = IFB200_ERR_INVALID_ARGUMENT;
    if (d.op < IFB200_CANVAS_FILL_RECT || d.op > IFB200_CANVAS_NORMALIZE_ALPHA) return fmt("unknown canvas op %llu", (unsigned)d.op);
    std::string e = check_window("canvas", d.px, d.w, d.h, d.stride);
    if (!e.empty()) return e;
    if (d.op == IFB200_CANVAS_FILL_RECT) {            // bitmaps.rs:1520-1533
        if (d.x2 == d.x1 || d.y2 == d.y1) return "";
        if (d.y2 <= d.y1 || d.x2 <= d.x1 || d.x2 > d.w || d.y2 > d.h)
            return fmt("rectangle %llu,%llu %llu,%llu must be within the window", d.x1, d.y1, d.x2, d.y2) + fmt(" (%llux%llu)", d.w, d.h);
        return "";
    }
    if (d.op == IFB200_CANVAS_NORMALIZE_ALPHA) return "";
    e = check_window("input", d.in, d.in_w, d.in_h, d.in_stride);
    if (!e.empty()) return e;
    if (d.op == IFB200_CANVAS_COPY_RECT) {            // copy_rect.rs:22-35 in 64 bits; a zero-size rectangle panics there (:68-79)
        const uint64_t fx = d.x1, fy = d.y1, tx = d.x2, ty = d.y2, cw = d.cw, ch = d.ch;
        if (d.in_w <= fx || d.in_h <= fy || d.in_w < fx + cw || d.in_h < fy + ch || d.w < tx + cw || d.h < ty + ch)
            return fmt("copy of %llux%llu from %llu,%llu", cw, ch, fx, fy) + fmt(" to %llu,%llu out of bounds", tx, ty);
        if (cw == 0 || ch == 0) return "zero-size copy";
    } else {                                          // clone_crop_fill_expand.rs:236-237; the copy of :246-253 needs in_w, in_h > 0
        if ((uint64_t)d.in_w + d.x1 + d.x2 != d.w || (uint64_t)d.in_h + d.y1 + d.y2 != d.h)
            return fmt("expanded canvas must be %llux%llu", (uint64_t)d.in_w + d.x1 + d.x2, (uint64_t)d.in_h + d.y1 + d.y2) +
                   fmt(", not %llux%llu", d.w, d.h);
        if (d.in_w == 0 || d.in_h == 0) return "empty input";
    }
    if (overlap(d)) return "input and canvas windows overlap";
    return "";
}

void canvas_plan(const ifb200_canvas_desc& d, CvWork& wk) {
    switch (d.op) {
    case IFB200_CANVAS_FILL_RECT:
        add(wk, kCvFill, 0, pack(d.color_bgra), d.px, d.stride, {d.x1, d.y1, d.x2 - d.x1, d.y2 - d.y1});
        break;
    case IFB200_CANVAS_NORMALIZE_ALPHA:               // bitmaps.rs:1570-1576
        if (!d.alpha_meaningful) add(wk, kCvOpaque, 0, 0, d.px, d.stride, {0, 0, d.w, d.h});
        break;
    case IFB200_CANVAS_COPY_RECT:
        plan_copy(d, d.alpha_meaningful != 0, d.in_alpha_meaningful != 0, d.x1, d.y1, d.x2, d.y2, d.cw, d.ch, wk);
        break;
    case IFB200_CANVAS_EXPAND: {                      // clone_crop_fill_expand.rs:239: the input's format for an opaque colour, else Bgra32
        const bool am = d.color_bgra[3] == 255 ? d.in_alpha_meaningful != 0 : true;
        std::vector<Rect> border;
        outside(d.w, d.h, {d.x1, d.y1, d.in_w, d.in_h}, border);
        for (const Rect& r : border) add(wk, kCvFill, 0, pack(d.color_bgra), d.px, d.stride, r);
        plan_copy(d, am, d.in_alpha_meaningful != 0, 0, 0, d.x1, d.y1, d.in_w, d.in_h, wk);
        break;
    }
    default: break;
    }
}

std::string canvas_prepare(const ifb200_canvas_desc* d, size_t n, CvWork& wk, int* code) {
    const std::string why = check_each("canvas", d, n, canvas_check, code);
    if (why.empty())
        for (size_t i = 0; i < n; ++i) canvas_plan(d[i], wk);
    return why;
}

}  // namespace ifb
