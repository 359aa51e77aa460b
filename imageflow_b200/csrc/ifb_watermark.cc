// ifb_watermark.cc -- see ifb_watermark.h.  Product code: must not include or link anything from the test oracle.
#include "ifb_watermark.h"

#include <algorithm>
#include <cstring>
#include <unordered_map>

#include "ifb_orient.h"   // groups_per_row
#include "ifb_prepare.h"

namespace ifb {
namespace {

// what F depends on (the resample of the watermark window as the library draws it)
struct Key {
    const uint8_t* in; uint32_t in_stride, in_w, in_h, am, op_bits, w, h; int32_t filter; uint32_t sharpen_bits, linear;
    bool operator==(const Key& o) const { return memcmp(this, &o, sizeof(Key)) == 0; }
};
struct KeyHash {
    size_t operator()(const Key& k) const {
        const uint32_t* p = reinterpret_cast<const uint32_t*>(&k);
        uint64_t x = 0x9E3779B97F4A7C15ull;
        for (size_t i = 0; i < sizeof(Key) / 4; ++i) x = (x ^ p[i]) * 0xC2B2AE3D27D4EB4Full;
        return (size_t)(x ^ (x >> 29));
    }
};

Key key_of(const ifb200_watermark_desc& d) {
    Key k;
    memset(&k, 0, sizeof k);                   // padding-free, but compared bytewise: zero it all the same
    float op = 1.0f;
    const bool applied = watermark_opacity(d.opacity, &op);
    const float sp = d.draw.sharpen_percent > 0.0f ? d.draw.sharpen_percent : 0.0f;
    k.in = d.draw.in; k.in_stride = d.draw.in_stride; k.in_w = d.draw.in_w; k.in_h = d.draw.in_h;
    k.am = (d.draw.alpha_meaningful || applied) ? 1u : 0u;
    k.op_bits = 0xFFFFFFFFu;                   // not a float the clamp can produce: no opacity step
    if (applied) memcpy(&k.op_bits, &op, 4);
    k.w = d.draw.w; k.h = d.draw.h; k.filter = d.draw.filter;
    memcpy(&k.sharpen_bits, &sp, 4);
    k.linear = d.draw.linear ? 1u : 0u;
    return k;
}

}  // namespace

std::string resample_check(const ifb200_resample_desc& d, int* code) {
    *code = IFB200_ERR_INVALID_ARGUMENT;
    if (!d.in || !d.canvas) return "null bitmap pointer";
    if ((uint64_t)d.h + d.y > d.cv_h || (uint64_t)d.w + d.x > d.cv_w)                     // scaling.rs:24-29
        return "Destination rectangle for scale2d is out of bounds";
    if (d.w == 0 || d.h == 0 || d.in_w == 0 || d.in_h == 0) return "empty bitmap";
    if (d.in_stride < d.in_w * 4ull || d.cv_stride < d.cv_w * 4ull || (d.in_stride & 3) || (d.cv_stride & 3))
        return "stride smaller than a BGRA row or not a multiple of 4";
    if (d.compose < 0 || d.compose > 2) return "unknown compositing mode " + std::to_string(d.compose);
    if (d.filter < 1 || d.filter > 31) {
        *code = IFB200_ERR_BAD_FILTER;
        return "unknown filter id " + std::to_string(d.filter);
    }
    return "";
}

bool watermark_opacity(float opacity, float* applied) {
    // f32::clamp(0, 1): NaN stays NaN, and NaN < 1 is false
    const float c = opacity != opacity ? opacity : std::min(std::max(opacity, 0.0f), 1.0f);
    *applied = c;
    return c < 1.0f;
}

std::string watermark_check(const ifb200_watermark_desc& d, int* code) {
    *code = IFB200_ERR_INVALID_ARGUMENT;
    if (d.draw.w == 0 || d.draw.h == 0) return "";
    const std::string why = resample_check(d.draw, code);
    if (!why.empty()) return why;
    if (d.draw.color_matrix) return "a watermark draw takes no colour matrix";
    if ((reinterpret_cast<uintptr_t>(d.draw.in) & 3) || (reinterpret_cast<uintptr_t>(d.draw.canvas) & 3))
        return "bitmap pointer not 4-byte aligned";
    if ((uint64_t)d.draw.w * d.draw.h > 0xffffffffull || (uint64_t)d.draw.in_w * d.draw.in_h > 0xffffffffull) return "window too large";
    return "";
}

void watermark_plan(const ifb200_watermark_desc* d, size_t n, const float* t_lin, const float* t_srgb, WmWork& wk) {
    std::unordered_map<Key, uint32_t, KeyHash> index;
    std::vector<std::vector<uint32_t>> members;       // descriptor indices of each group, in call order
    Key last{}; uint32_t last_g = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; ++i) {
        if (d[i].draw.w == 0 || d[i].draw.h == 0) continue;
        const Key k = key_of(d[i]);
        if (last_g == 0xFFFFFFFFu || !(k == last)) {   // consecutive jobs of one watermark cost one compare, not a lookup
            auto it = index.find(k);
            if (it == index.end()) {
                it = index.emplace(k, (uint32_t)members.size()).first;
                members.emplace_back();
                wk.rep.push_back((uint32_t)i);
                float op = 1.0f;
                wk.opacity.push_back(watermark_opacity(d[i].opacity, &op) ? op : 1.0f);
            }
            last = k; last_g = it->second;
        }
        members[last_g].push_back((uint32_t)i);
    }
    uint64_t first = 0;
    for (size_t g = 0; g < members.size(); ++g) {
        const ifb200_watermark_desc& r = d[wk.rep[g]];
        WmGroup gr{};
        gr.f = reinterpret_cast<const float*>((uintptr_t)wk.f_bytes);
        gr.w = r.draw.w; gr.h = r.draw.h;
        gr.rows = std::min<uint32_t>(gr.h, std::max<uint32_t>(1u, kWmTilePixels / gr.w));
        gr.tiles = (gr.h + gr.rows - 1) / gr.rows;
        gr.job0 = (uint32_t)wk.jobs.size(); gr.n = (uint32_t)members[g].size();
        gr.first = (uint32_t)std::min<uint64_t>(first, 0xffffffffull);
        first += (uint64_t)gr.tiles * gr.n;
        wk.f_bytes += (uint64_t)gr.w * gr.h * 16u;
        wk.groups.push_back(gr);
        const bool applied = wk.opacity[g] < 1.0f;
        for (uint32_t i : members[g]) {
            const ifb200_resample_desc& dd = d[i].draw;
            WmJob j{};
            j.out = dd.canvas + (size_t)dd.y * dd.cv_stride + (size_t)dd.x * 4;
            j.stride = dd.cv_stride;
            j.groups = groups_per_row(j.out, j.stride, dd.w);
            const bool am = dd.alpha_meaningful || applied;                 // the Alpha filter makes the copy Bgra32
            const int32_t compose = dd.compose == IFB200_REPLACE_SELF ? IFB200_BLEND_WITH_SELF : dd.compose;   // scale_render.rs:282-284
            j.flags = (dd.linear ? 1u : 0u) | (am ? 2u : 0u) | ((uint32_t)compose << 2);                    // JF_LINEAR, JF_ALPHA, compose
            if (compose == IFB200_BLEND_WITH_MATTE && am) {                 // as make_job (ifb_engine.cu)
                const float* T = dd.linear ? t_lin : t_srgb;
                const float ma = (float)dd.matte_bgra[3] * (1.0f / 255.0f);
                j.matte[0] = T[dd.matte_bgra[0]] * ma; j.matte[1] = T[dd.matte_bgra[1]] * ma; j.matte[2] = T[dd.matte_bgra[2]] * ma; j.matte[3] = ma;
            }
            wk.jobs.push_back(j);
        }
    }
}

std::string watermark_prepare(const ifb200_watermark_desc* d, size_t n, const float* t_lin, const float* t_srgb, WmWork& wk, int* code) {
    const std::string why = check_each("watermark", d, n, watermark_check, code);
    if (why.empty()) watermark_plan(d, n, t_lin, t_srgb, wk);
    return why;
}

}  // namespace ifb
