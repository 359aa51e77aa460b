// ifb_color.cc -- see ifb_color.h.  Product code: must not include or link anything from the test oracle.  Compiled with
// -ffp-contract=off: the table entries are the reference's f32 sums, without fused multiply-adds.
#include "ifb_color.h"

#include <algorithm>

#include "ifb_orient.h"   // groups_per_row
#include "ifb_prepare.h"

namespace ifb {
namespace {

// the channel (r, g, b, a = 0..3, the matrix's index order) stored at byte position k of a BGRA pixel
constexpr int kChannelAt[4] = {2, 1, 0, 3};

// ColorMatrixSrgb with m[k][c] == 0 for every input k != c (k, c < 4): each output byte depends on its own input byte only.  The test
// is exact zero, so NaN and infinity never qualify.
bool separable(const float* m) {
    for (int k = 0; k < 4; ++k)
        for (int c = 0; c < 4; ++c)
            if (k != c && m[k * 5 + c] != 0.0f) return false;
    return true;
}

// output channel c of color_matrix.rs:21-24 for a pixel whose channel c is v and whose other channels are 0.  For a separable matrix
// this is exact for any pixel: a zero coefficient times a finite non-negative byte is a zero of the coefficient's sign either way.
uint8_t matrix_entry(const float* m, int c, uint32_t v) {
    float x[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    x[c] = (float)v;
    const float bias = m[4 * 5 + c] * 255.0f;
    return color_clamp(m[0 * 5 + c] * x[0] + m[1 * 5 + c] * x[1] + m[2 * 5 + c] * x[2] + m[3 * 5 + c] * x[3] + bias);
}

void add(std::vector<ClJob>& jobs, std::vector<uint32_t>& first, const ClJob& job, uint64_t ctas) {
    if (first.empty()) first.push_back(0);
    jobs.push_back(job);
    first.push_back((uint32_t)std::min<uint64_t>(first.back() + ctas, 0xffffffffull));
}

// appends a planned job, and its histogram job when it white-balances
void add_job(ClWork& wk, ClJob j) {
    const uint64_t ctas = ((uint64_t)j.groups * j.h + kClCtaGroups - 1) / kClCtaGroups;
    if (j.wb_seg < j.nseg) {
        j.wb = (uint32_t)wk.wb_jobs.size();
        ClJob hj = j;
        hj.nseg = j.wb_seg;
        add(wk.wb_jobs, wk.wb_first, hj, ctas);
    }
    add(wk.jobs, wk.first, j, ctas);
}

}  // namespace

uint8_t color_clamp(float clr) {                          // (clr as f64 + 0.5) as i16 as u16, then > 255 -> 0 or 255
    if (clr != clr) return 0;
    const double v = (double)clr + 0.5;
    const int32_t i = v >= 32767.0 ? 32767 : v <= -32768.0 ? -32768 : (int32_t)v;
    uint16_t r = (uint16_t)(int16_t)i;
    if (r > 255) r = clr < 0.0f ? 0 : 255;
    return (uint8_t)r;
}

size_t ClWork::bytes() const {
    return (jobs.size() + wb_jobs.size()) * sizeof(ClJob) + (first.size() + wb_first.size()) * sizeof(uint32_t) + segs.size() * sizeof(ClSeg) +
           tables.size() + mats.size() * sizeof(float);
}

std::string color_check(const ifb200_color_desc& d, int* code) {
    *code = IFB200_ERR_INVALID_ARGUMENT;
    if (d.w == 0 || d.h == 0 || d.n_steps == 0) return "";
    if (d.n_steps > kClMaxSteps) return "more than " + std::to_string(kClMaxSteps) + " steps";
    if (!d.steps) return "null steps pointer";
    if (!d.px) return "null bitmap pointer";
    if (reinterpret_cast<uintptr_t>(d.px) & 3) return "bitmap pointer not 4-byte aligned";
    if (d.stride < d.w * 4ull || (d.stride & 3)) return "stride smaller than a BGRA row or not a multiple of 4";
    if ((uint64_t)d.w * d.h > 0xffffffffull) return "window too large";
    int wb = 0;
    for (uint32_t i = 0; i < d.n_steps; ++i) {
        const ifb200_color_step& s = d.steps[i];
        if (s.kind == IFB200_COLOR_WHITE_BALANCE) {
            if (s.threshold != s.threshold) return "step " + std::to_string(i) + ": white balance threshold is NaN";
            if (++wb > 1) {
                *code = IFB200_ERR_NOT_IMPLEMENTED;
                return "step " + std::to_string(i) + ": a second white balance in one job";
            }
        } else if (s.kind != IFB200_COLOR_MATRIX && s.kind != IFB200_COLOR_ENABLE_TRANSPARENCY) {
            return "step " + std::to_string(i) + ": unknown step kind " + std::to_string(s.kind);
        }
    }
    return "";
}

void color_plan(const ifb200_color_desc& d, ClWork& wk) {
    if (d.w == 0 || d.h == 0 || d.n_steps == 0) return;
    ClJob j{};
    const int32_t am_in = d.alpha_meaningful != 0;
    const bool reuse = wk.last_steps == d.steps && wk.last_n == d.n_steps && wk.last_am == am_in;
    if (reuse) j = wk.last;
    j.px = d.px; j.w = d.w; j.h = d.h; j.stride = d.stride;
    j.groups = groups_per_row(d.px, d.stride, d.w);
    if (reuse) {
        if (j.nseg == 0) return;
        add_job(wk, j);
        return;
    }
    j.seg0 = (uint32_t)wk.segs.size(); j.tab0 = (uint32_t)(wk.tables.size() / 1024); j.mat0 = (uint32_t)(wk.mats.size() / 20);
    j.wb = kClNone; j.wb_seg = kClNone;
    bool am = am_in != 0;
    bool open = false;                                 // the last segment is a kClTable that the next separable step composes into
    auto new_table = [&](uint32_t kind) {
        const size_t t = wk.tables.size();
        wk.tables.resize(t + 1024);
        for (uint32_t k = 0; k < 4; ++k)
            for (uint32_t v = 0; v < 256; ++v) wk.tables[t + k * 256 + v] = (uint8_t)v;
        wk.segs.push_back({kind, j.ntab++});
        return t;
    };
    auto table = [&]() -> uint8_t* {                   // the open table, opened when there is none
        if (!open) new_table(kClTable);
        open = true;
        return &wk.tables[wk.tables.size() - 1024];
    };
    for (uint32_t i = 0; i < d.n_steps; ++i) {
        const ifb200_color_step& s = d.steps[i];
        if (s.kind == IFB200_COLOR_MATRIX) {
            const float* m = s.matrix;
            if (separable(m)) {
                uint8_t* t = table();
                for (int k = 0; k < 4; ++k) {
                    uint8_t step[256];
                    for (uint32_t v = 0; v < 256; ++v) step[v] = matrix_entry(m, kChannelAt[k], v);
                    for (uint32_t v = 0; v < 256; ++v) t[k * 256 + v] = step[t[k * 256 + v]];
                }
            } else {
                for (int c = 0; c < 4; ++c) {
                    for (int k = 0; k < 4; ++k) wk.mats.push_back(m[k * 5 + c]);
                    wk.mats.push_back(m[4 * 5 + c] * 255.0f);       // color_matrix.rs:9-12
                }
                wk.segs.push_back({kClMatrix, j.nmat++});
                open = false;
            }
        } else if (s.kind == IFB200_COLOR_ENABLE_TRANSPARENCY) {
            if (!am) {                                  // Bgr32: A = 255 and Bgra32 from here on; Bgra32: the node deletes itself
                uint8_t* t = table();
                for (uint32_t v = 0; v < 256; ++v) t[3 * 256 + v] = 255;
                am = true;
            }
        } else {                                        // IFB200_COLOR_WHITE_BALANCE (color_check admits no other kind)
            j.wb_seg = (uint32_t)(wk.segs.size() - j.seg0);
            new_table(kClWb);
            open = false;
            j.low = (double)(s.threshold < 0.0f ? 0.006f : s.threshold);    // white_balance.rs:76-77, f64::from(f32)
        }
    }
    j.nseg = (uint32_t)(wk.segs.size() - j.seg0);
    if (j.wb_seg == kClNone) {                         // shareable with the next job of the same chain
        j.wb_seg = j.nseg;
        wk.last_steps = d.steps; wk.last_n = d.n_steps; wk.last_am = am_in; wk.last = j;
    } else {
        wk.last_steps = nullptr;
    }
    if (j.nseg == 0) return;                           // nothing but EnableTransparency on Bgra32: no pixel changes
    add_job(wk, j);
}

std::string color_prepare(const ifb200_color_desc* d, size_t n, ClWork& wk, int* code) {
    const std::string why = check_each("color", d, n, color_check, code);
    if (why.empty())
        for (size_t i = 0; i < n; ++i) color_plan(d[i], wk);
    return why;
}

}  // namespace ifb
