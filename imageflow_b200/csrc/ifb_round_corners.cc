// ifb_round_corners.cc -- see ifb_round_corners.h.  Product code: must not include or link anything from the test oracle.
//
// Every float below is computed in f32 in the reference's operation order (the library is built with -ffp-contract=off, so
// nothing is fused); the kernel redoes the per-row and per-pixel parts on the GPU from the fields planned here.
#include "ifb_round_corners.h"

#include <algorithm>
#include <cmath>

#include "../../include/ifb200.h"
#include "ifb_prepare.h"

namespace ifb {
namespace {

// Rust's `f32 as usize` (saturating; NaN -> 0), kept in 64 bits
uint64_t as_usize(float f) {
    if (!(f > 0.0f)) return 0;
    if (f >= 18446744073709551616.0f) return UINT64_MAX;
    return (uint64_t)f;
}
// f32::clamp: NaN stays NaN
float clampf(float v, float lo, float hi) {
    if (v < lo) v = lo;
    if (v > hi) v = hi;
    return v;
}

struct QuadrantInfo { uint32_t x, y, width, height; float radius, cx, cy; bool is_top, is_left; };

// plan_quadrants (rounded_corners.rs:41-159) for RoundCornersRadius::Custom([top_left, top_right, bottom_left, bottom_right])
void plan_custom(const float r[4], uint32_t w, uint32_t h, QuadrantInfo q[4]) {
    const uint32_t right_half_width = w / 2, bottom_half_height = h / 2;
    const uint32_t left_half_width = w - right_half_width, top_half_height = h - bottom_half_height;
    q[0] = {0, 0, left_half_width, top_half_height, r[0], r[0], r[0], true, true};
    q[1] = {left_half_width, 0, right_half_width, top_half_height, r[1], (float)w - r[1], r[1], true, false};
    q[2] = {0, top_half_height, left_half_width, bottom_half_height, r[2], r[2], (float)h - r[2], false, true};
    q[3] = {left_half_width, top_half_height, right_half_width, bottom_half_height, r[3], (float)w - r[3], (float)h - r[3], false, false};
}

// The job of a valid, non-empty descriptor.  get_radius (rounded_corners.rs:5-33): its Custom array is [tl, tr, bl, br]; d.radius
// is in the field order of RoundCornersMode::*Custom [tl, tr, br, bl].
RcJob plan_job(const ifb200_round_corners_desc& d) {
    const uint32_t w = d.w, h = d.h;
    const float* radius = d.radius;
    const float smallest = (float)std::min(w, h);
    auto pct = [&](float p) { return smallest * clampf(p, 0.0f, 100.0f) / 200.0f; };
    auto pix = [&](float p) { return clampf(p, 0.0f, smallest / 2.0f); };
    QuadrantInfo q[4];
    switch (d.mode) {
    case IFB200_CORNERS_PERCENTAGE: { const float v = pct(radius[0]); const float r[4] = {v, v, v, v}; plan_custom(r, w, h, q); break; }
    case IFB200_CORNERS_PIXELS: { const float v = pix(radius[0]); const float r[4] = {v, v, v, v}; plan_custom(r, w, h, q); break; }
    case IFB200_CORNERS_PERCENTAGE_CUSTOM: {
        const float r[4] = {pct(radius[0]), pct(radius[1]), pct(radius[3]), pct(radius[2])};
        plan_custom(r, w, h, q); break;
    }
    case IFB200_CORNERS_PIXELS_CUSTOM: {
        const float r[4] = {pix(radius[0]), pix(radius[1]), pix(radius[3]), pix(radius[2])};
        plan_custom(r, w, h, q); break;
    }
    default: {                                                   // IFB200_CORNERS_CIRCLE, :46-64: the quadrants of the centred square, moved
        const uint32_t s = std::min(w, h);
        const uint32_t off_x = (uint32_t)(std::max<int64_t>((int64_t)w - (int64_t)h, 0) / 2);
        const uint32_t off_y = (uint32_t)(std::max<int64_t>((int64_t)h - (int64_t)w, 0) / 2);
        const float v = smallest / 2.0f;
        const float r[4] = {v, v, v, v};
        plan_custom(r, s, s, q);
        for (auto& e : q) { e.x += off_x; e.y += off_y; e.cx += (float)off_x; e.cy += (float)off_y; }
        break;
    }
    }

    const float volumetric_offset = 0.56419f;                 // :200-202
    RcJob job{};
    job.px = d.px; job.stride = d.stride;
    job.matte = (uint32_t)d.matte_bgra[0] | ((uint32_t)d.matte_bgra[1] << 8) | ((uint32_t)d.matte_bgra[2] << 16) | ((uint32_t)d.matte_bgra[3] << 24);
    job.w = w; job.h = h;
    job.top_rows = q[0].y;                                   // :209-212 (q[0].y > 0 only for CIRCLE on a tall frame)
    job.bottom_from = std::min(h, q[2].y + q[2].height);     // :213-216
    for (int i = 0; i < 4; ++i) {
        const QuadrantInfo& a = q[i];
        RcQuad& o = job.q[i];
        const uint32_t bottom = a.y + a.height, right = a.x + a.width;
        const uint64_t radius_ceil = as_usize(std::ceil(a.radius));
        // :218-227; the clamps only matter where the reference would index out of bounds
        const uint64_t start_y = a.is_top ? a.y : (radius_ceil > bottom ? 0 : bottom - radius_ceil);
        const uint64_t end_y = a.is_top ? std::min<uint64_t>((uint64_t)a.y + radius_ceil, h) : bottom;
        o.cx = a.cx; o.cy = a.cy;
        o.roi = a.radius + (1.0f - volumetric_offset);
        o.ros = a.radius - volumetric_offset;
        o.raw = o.roi - o.ros;
        o.roi2 = o.roi * o.roi;
        o.ros2 = o.ros * o.ros;
        o.y = a.y; o.bottom = bottom;
        o.start_y = (uint32_t)start_y; o.end_y = (uint32_t)std::max(end_y, start_y);
        o.clear_from = a.is_left ? 0u : right;
        o.clear_to = a.is_left ? a.x : w;
        o.is_left = a.is_left ? 1u : 0u;
    }
    return job;
}

}  // namespace

std::string round_corners_check(const ifb200_round_corners_desc& d, int* code) {
    if (code) *code = IFB200_ERR_INVALID_ARGUMENT;
    if (d.mode < IFB200_CORNERS_PERCENTAGE || d.mode > IFB200_CORNERS_PIXELS_CUSTOM) return "unknown corners mode " + std::to_string(d.mode);
    if (d.w == 0 || d.h == 0) return "";
    if (!d.px) return "null bitmap pointer";
    if (d.stride < d.w * 4ull || (d.stride & 3)) return "stride smaller than a BGRA row or not a multiple of 4";
    if ((uint64_t)d.w * d.h > 0xffffffffull) return "bitmap too large";
    return "";
}

void round_corners_plan(const ifb200_round_corners_desc& d, RcWork& wk, std::vector<RcRect>* rects) {
    if (d.w == 0 || d.h == 0) return;
    const RcJob job = plan_job(d);
    std::vector<RcRect> cover;
    round_corners_cover(job, cover);
    const uint32_t j = (uint32_t)wk.jobs.size();
    wk.jobs.push_back(job);
    for (const RcRect& r : cover) {
        const uint64_t area = (uint64_t)r.w * r.h;
        for (uint64_t f = 0; f < area; f += kRcTilePixels)
            wk.tiles.push_back({j, r.x0, r.y0, r.w, (uint32_t)f, (uint32_t)std::min<uint64_t>(kRcTilePixels, area - f)});
    }
    if (rects) rects->insert(rects->end(), cover.begin(), cover.end());
}

std::string round_corners_prepare(const ifb200_round_corners_desc* d, size_t n, RcWork& wk, int* code) {
    const std::string why = check_each("round corners", d, n, round_corners_check, code);
    if (why.empty())
        for (size_t i = 0; i < n; ++i) round_corners_plan(d[i], wk);
    return why;
}

void round_corners_cover(const RcJob& job, std::vector<RcRect>& out) {
    const uint32_t w = job.w, h = job.h;
    // every step as (rows [y0, y1), prefix [0, left) or suffix [right, w), whether it may blend)
    struct Step { uint32_t y0, y1, left, right; bool blend; };
    std::vector<Step> steps;
    if (job.top_rows > 0) steps.push_back({0, std::min(job.top_rows, h), w, 0, false});
    if (job.bottom_from < h) steps.push_back({job.bottom_from, h, w, 0, false});
    for (const RcQuad& q : job.q) {
        const bool left = q.is_left != 0;
        if (q.clear_from != q.clear_to) {                    // :242-250
            const uint32_t l = left ? q.clear_to : 0, r = left ? w : q.clear_from;
            if (q.y < std::min(q.start_y, q.bottom)) steps.push_back({q.y, std::min(q.start_y, q.bottom), l, r, false});
            if (q.end_y < q.bottom) steps.push_back({q.end_y, q.bottom, l, r, false});
        }
        if (q.start_y < q.end_y) {
            // Row edges (:276-286) lie within [0, ceil(cx)) for a left quadrant and [floor(cx), w) for a right one: cx - d rounds
            // to at most cx and cx + d to at least cx for d >= 0, and floor / ceil / max / min are monotonic.
            const uint32_t l = left ? (uint32_t)std::min<uint64_t>(as_usize(std::ceil(q.cx)), w) : 0;
            const uint32_t r = left ? w : (uint32_t)std::min<uint64_t>(as_usize(std::floor(q.cx)), w);
            steps.push_back({q.start_y, q.end_y, l, r, true});
        }
    }
    std::vector<uint32_t> cuts{0, h};
    for (const Step& s : steps) { cuts.push_back(s.y0); cuts.push_back(s.y1); }
    std::sort(cuts.begin(), cuts.end());
    cuts.erase(std::unique(cuts.begin(), cuts.end()), cuts.end());
    struct Band { uint32_t y0, y1, left, right; bool blend_l, blend_r; };
    std::vector<Band> bands;
    for (size_t i = 0; i + 1 < cuts.size(); ++i) {
        Band b{cuts[i], cuts[i + 1], 0, w, false, false};
        for (const Step& s : steps) {
            if (s.y0 > b.y0 || s.y1 < b.y1) continue;        // steps start and end on cuts: either covers the band or misses it
            if (s.left > 0) { b.left = std::max(b.left, s.left); b.blend_l |= s.blend; }
            if (s.right < w) { b.right = std::min(b.right, s.right); b.blend_r |= s.blend; }
        }
        if (b.left == 0 && b.right == w) continue;
        if (!bands.empty() && bands.back().y1 == b.y0 && bands.back().left == b.left && bands.back().right == b.right &&
            bands.back().blend_l == b.blend_l && bands.back().blend_r == b.blend_r) { bands.back().y1 = b.y1; continue; }
        bands.push_back(b);
    }
    for (const Band& b : bands) {
        const uint32_t rows = b.y1 - b.y0;
        if (b.left >= b.right) { out.push_back({0, b.y0, w, rows, !(b.blend_l || b.blend_r)}); continue; }
        if (b.left > 0) out.push_back({0, b.y0, b.left, rows, !b.blend_l});
        if (b.right < w) out.push_back({b.right, b.y0, w - b.right, rows, !b.blend_r});
    }
}

}  // namespace ifb
