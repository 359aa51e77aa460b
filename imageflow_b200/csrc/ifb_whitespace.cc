// ifb_whitespace.cc -- see ifb_whitespace.h.  Product code: must not include or link anything from oracle/.
//
// Why a replay and not a reduction: the reference never looks at all pixels.  Its scan rectangle for the whole image ends at
// floor(1.0 * (w - 1)) (whitespace.rs:221-236), windows of at most 2048 grayscale bytes overlap by two, and every window is
// skipped, shrunk or moved according to the bounding box found so far (:352-408).  The bounding box of all codes is an outer
// bound of the result and differs from it on about one image in seven (measured in the tests), so the walk is
// reproduced step by step.  detect_content_from_codes is that walk over a code map, on the host (the public
// ifb200_detect_content_from_codes, and the reference the tests hold the device walk to); whitespace_grid / detect_content_prepare
// plan the device walk of ifb200_batch_detect_content_many (ifb_whitespace.h, DESIGN.md §5.16).
#include "ifb_whitespace.h"

#include <algorithm>
#include <cmath>
#include <cstring>

#include "ifb_prepare.h"

namespace ifb {
namespace {

enum class Edge { Top, Right, Bottom, Left, None };
struct Region { Edge edge; float x1, y1, x2, y2; };          // fractions of (w - 1), (h - 1)

// whitespace.rs:30-131: twelve thin strips.  Each has x1 == x2 or y1 == y2 and is rejected by the emptiness test of
// search_rect() before it is widened (:256-258) -- kept here because the reference walks them.
constexpr Region kQuick[12] = {
    {Edge::Left, 0.f, .5f, .5f, .5f},     {Edge::Right, .5f, .5f, 1.f, .5f},     {Edge::Left, 0.f, .677f, .5f, .677f}, {Edge::Right, .5f, .677f, 1.f, .677f},
    {Edge::Left, 0.f, .333f, .5f, .333f}, {Edge::Right, .5f, .333f, 1.f, .333f}, {Edge::Top, .5f, 0.f, .5f, .5f},      {Edge::Top, .677f, 0.f, .677f, .5f},
    {Edge::Top, .333f, 0.f, .333f, .5f},  {Edge::Bottom, .5f, .5f, .5f, 1.f},    {Edge::Bottom, .677f, .5f, .677f, 1.f}, {Edge::Bottom, .333f, .5f, .333f, 1.f}};
constexpr Region kInward[4] = {{Edge::Top, 0.f, 0.f, 1.f, 1.f}, {Edge::Right, 0.f, 0.f, 1.f, 1.f}, {Edge::Bottom, 0.f, 0.f, 1.f, 1.f}, {Edge::Left, 0.f, 0.f, 1.f, 1.f}};
constexpr Region kFull = {Edge::None, 0.f, 0.f, 1.f, 1.f};
constexpr uint32_t kBuffer = 2048;                           // the reference's grayscale window, in pixels

struct Walk {
    const uint8_t* codes; uint32_t w, h;
    uint32_t lo_x, hi_x, lo_y, hi_y;                         // bounding box so far: min_x, max_x, min_y, max_y
    uint64_t visited = 0;

    struct Box { uint32_t x1, y1, x2, y2; bool any; };
    Box search_rect(const Region& r) const {                 // whitespace.rs:220-281
        auto at = [](float f, uint32_t n) { return std::min(n, (uint32_t)std::floor(f * (float)(n - 1))); };
        uint32_t x1 = at(r.x1, w), x2 = at(r.x2, w), y1 = at(r.y1, h), y2 = at(r.y2, h);
        if (r.edge == Edge::Left) { x1 = 0; x2 = std::min(x2, lo_x); }
        else if (r.edge == Edge::Right) { x1 = std::max(x1, hi_x); x2 = w; }
        else if (r.edge == Edge::Top) { y1 = 0; y2 = std::min(y2, lo_y); }
        else if (r.edge == Edge::Bottom) { y1 = std::max(y1, hi_y); y2 = h; }
        if (x1 == x2 || y1 == y2) return {0, 0, 0, 0, false};
        const bool horizontal = r.edge == Edge::Left || r.edge == Edge::Right, vertical = r.edge == Edge::Top || r.edge == Edge::Bottom;
        const uint32_t need_w = horizontal ? 3u : 7u, need_h = vertical ? 3u : 7u;
        while (y2 - y1 < need_h && (y1 > 0 || y2 < h)) { if (y1) --y1; y2 = std::min(h, y2 + 1); }
        while (x2 - x1 < need_w && (x1 > 0 || x2 < w)) { if (x1) --x1; x2 = std::min(w, x2 + 1); }
        return {x1, y1, x2, y2, true};
    }

    void window(uint32_t bx, uint32_t by, uint32_t bw, uint32_t bh) {        // sobel_scharr_detect over the window's interior
        // The window only takes minima and maxima over its edge pixels, so the order inside it is free: runs of kNoEdge (blank
        // paper, the common case) are skipped eight codes at a time.
        if (bw < 3 || bh < 3) return;
        const uint32_t xa = bx + 1, xb = bx + bw - 1;        // interior columns [xa, xb)
        visited += (uint64_t)(xb - xa) * (bh - 2);
        for (uint32_t y = by + 1; y + 1 < by + bh; ++y) {
            const uint8_t* row = codes + (size_t)y * w;
            auto take = [&](uint32_t x) {
                const uint32_t c = row[x];
                if (c == kNoEdge) return;
                lo_x = std::min(lo_x, x - 1 + (c & 3u));
                hi_x = std::max(hi_x, x + ((c >> 2) & 3u));                  // (x - 1) + (stored + 1)
                lo_y = std::min(lo_y, y - 1 + ((c >> 4) & 3u));
                hi_y = std::max(hi_y, y + ((c >> 6) & 3u));
            };
            uint32_t x = xa;
            for (; x + 8 <= xb; x += 8) {
                uint64_t v;
                std::memcpy(&v, row + x, 8);
                if (v != ~0ull) for (uint32_t k = 0; k < 8; ++k) take(x + k);
            }
            for (; x < xb; ++x) take(x);
        }
    }

    void region(const Region& r) {                           // whitespace.rs:333-421
        const Box s = search_rect(r);
        if (!s.any) return;
        const uint32_t rw = s.x2 - s.x1, rh = s.y2 - s.y1;
        const uint32_t ww = std::min(rw, r.edge == Edge::None ? kBuffer / 7u : (uint32_t)std::ceil(std::sqrt((float)kBuffer)));
        const uint32_t wh = std::min(rh, kBuffer / ww);
        if (ww <= 2 || wh <= 2) return;                      // the reference would divide by zero; detect_content never gets here
        const uint32_t rows = (uint32_t)std::ceil((float)rh / (float)(wh - 2)), cols = (uint32_t)std::ceil((float)rw / (float)(ww - 2));
        for (uint32_t j = 0; j < rows; ++j) {
            for (uint32_t i = 0; i < cols; ++i) {
                uint32_t bx = s.x1 + (ww - 2) * i, by = s.y1 + (wh - 2) * j;
                uint32_t bw = std::min(std::max(3u, s.x2 - bx), ww), bh = std::min(std::max(3u, s.y2 - by), wh);
                const uint32_t ex = bx + bw, ey = by + bh;
                const bool in_x = lo_x < bx && hi_x > ex, in_y = lo_y < by && hi_y > ey;      // already inside the box on that axis
                if (in_x && in_y) continue;
                if (in_y && lo_x < ex && ex < hi_x) bw = std::max(3u, lo_x - bx);
                else if (in_y && hi_x > bx && bx > lo_x) { bx = std::min(ex - 3, hi_x); bw = ex - bx; }
                if (in_x && lo_y < ey && ey < hi_y) bh = std::max(3u, lo_y - by);
                else if (in_x && hi_y > by && by > lo_y) { by = std::min(ey - 3, hi_y); bh = ey - by; }
                if (by + bh > h) { if (bh <= h) by = h - bh; else { by = 0; bh = h; } }
                if (bx + bw > w) { if (bw <= w) bx = w - bw; else { bx = 0; bw = w; } }
                window(bx, by, bw, bh);
            }
        }
    }
};

}  // namespace

bool detect_content_from_codes(const uint8_t* codes, uint32_t w, uint32_t h, uint32_t rect[4], uint64_t* centres) {
    if (!codes || !rect || w == 0 || h == 0 || w > 0x7fffffffu || h > 0x7fffffffu) return false;
    if (centres) *centres = 0;
    rect[0] = 0; rect[1] = 0; rect[2] = w; rect[3] = h;
    if (w < 3 || h < 3) return true;                         // whitespace.rs:288-290
    Walk k{codes, w, h, w, 0, h, 0};
    for (const Region& r : kQuick) k.region(r);
    const int64_t outside = (int64_t)k.lo_x * h + (int64_t)k.lo_y * w + ((int64_t)w - k.hi_x) * h + ((int64_t)h - k.hi_y) * w;
    if (outside > (int64_t)h * w) k.region(kFull);           // :312-320
    else for (const Region& r : kInward) k.region(r);
    if (!(k.lo_x == w && k.hi_x == 0 && k.lo_y == h && k.hi_y == 0)) { rect[0] = k.lo_x; rect[1] = k.lo_y; rect[2] = k.hi_x; rect[3] = k.hi_y; }
    if (centres) *centres = k.visited;
    return true;
}

void whitespace_grid(uint32_t w, uint32_t h, WsJob& job, std::vector<WsColumn>& cols) {
    job.rows = 0; job.ncols = 0;
    const Walk k{nullptr, w, h, w, 0, h, 0};
    const Walk::Box s = k.search_rect(kFull);                // the full scan reads no box (Edge::None)
    if (!s.any) return;
    // Walk::region's arithmetic, for the full scan
    const uint32_t rw = s.x2 - s.x1, rh = s.y2 - s.y1;
    const uint32_t ww = std::min(rw, kBuffer / 7u), wh = std::min(rh, kBuffer / ww);
    if (ww <= 2 || wh <= 2) return;
    job.y1 = s.y1; job.y2 = s.y2; job.wh = wh;
    job.rows = (uint32_t)std::ceil((float)rh / (float)(wh - 2));
    job.ncols = (uint32_t)std::ceil((float)rw / (float)(ww - 2));
    for (uint32_t i = 0; i < job.ncols; ++i) {
        uint32_t bx = s.x1 + (ww - 2) * i, bw = std::min(std::max(3u, s.x2 - bx), ww);
        WsColumn c{bx, bx + bw, 0, 0, 0, 0};
        if (bx + bw > w) { if (bw <= w) bx = w - bw; else { bx = 0; bw = w; } }
        c.xa = bx + 1; c.xb = std::max(bx + 1, bx + bw - 1);
        cols.push_back(c);
    }
}

std::string detect_content_check(const ifb200_detect_content_desc& d, int* code) {
    if (code) *code = IFB200_ERR_INVALID_ARGUMENT;
    // whitespace_check's limits and messages (ifb_engine.cu), plus the alignment of the kernels' 4-byte pixel loads
    if (!d.px) return "null bitmap pointer";
    if (d.w == 0 || d.h == 0) return "empty bitmap";
    if (d.stride < d.w * 4ull || (d.stride & 3)) return "stride smaller than a BGRA row or not a multiple of 4";
    if (reinterpret_cast<uintptr_t>(d.px) & 3) return "bitmap pointer not 4-byte aligned";
    if (d.w > 0x7fffffffu || d.h > 0x7fffffffu) return "oversized bitmap";
    if (d.threshold > 0x7fffffffu) return "threshold out of range";
    return "";
}

std::string detect_content_prepare(const ifb200_detect_content_desc* d, size_t n, WsWork& wk, int* code, uint32_t* rects, uint64_t* visited) {
    const std::string why = check_each("detect_content", d, n, detect_content_check, code);
    if (!why.empty()) return why;
    for (size_t i = 0; i < n; ++i) {
        if (rects) { rects[4 * i] = 0; rects[4 * i + 1] = 0; rects[4 * i + 2] = d[i].w; rects[4 * i + 3] = d[i].h; }
        if (visited) visited[i] = 0;
        if (d[i].w < 3 || d[i].h < 3) continue;              // whitespace.rs:288-290
        WsJob job{};
        job.w = d[i].w; job.h = d[i].h; job.col0 = (uint32_t)wk.cols.size();
        whitespace_grid(job.w, job.h, job, wk.cols);
        job.sum0 = wk.n_sums;
        const uint64_t bands = (job.h + kWsBand - 1) / kWsBand;
        for (uint32_t c = job.col0; c < job.col0 + job.ncols; ++c) {
            WsColumn& col = wk.cols[c];
            col.chunk0 = job.tch; col.nch = (col.xb - col.xa + kWsChunk - 1) / kWsChunk;
            job.tch += col.nch;
        }
        for (uint32_t c = job.col0; c < job.col0 + job.ncols; ++c) {
            const WsColumn& col = wk.cols[c];
            if (col.nch == 0) continue;
            wk.segs.push_back({d[i].px, job.w, job.h, d[i].stride, d[i].alpha_meaningful ? 1u : 0u, (int32_t)d[i].threshold, col.xa, col.xb,
                               col.chunk0, col.nch, job.tch, job.sum0});
            if (wk.first.empty()) wk.first.push_back(0);
            wk.first.push_back((uint32_t)std::min<uint64_t>(wk.first.back() + bands * col.nch, 0xffffffffull));
        }
        wk.n_sums += (uint64_t)job.h * job.tch;
        wk.jobs.push_back(job);
        wk.job_of.push_back((uint32_t)i);
    }
    return "";
}

}  // namespace ifb
