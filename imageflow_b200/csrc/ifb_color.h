// ifb_color.h -- host planner of ifb200_batch_color_chain (include/ifb200.h: a chain of colour nodes as one pass per frame).  Product
// code, plain C++ without CUDA calls (tests/cpu_emu links it unchanged): validation of each descriptor, and each job's steps compiled
// into segments that the kernels of ifb_color_kernel.cuh evaluate per pixel in registers:
//   kClTable   a maximal run of channel-separable steps, composed into one 4 x 256 byte table (by byte position: B, G, R, A);
//   kClMatrix  a step that mixes channels, kept as 20 floats in the order the kernel reads them (out c: m[k][c] for k = r, g, b, a,
//              then the bias m[4][c] * 255), as color_matrix_locked uploads them;
//   kClWb      the white balance: a table too, whose R, G, B entries the maps kernel fills on the device after the histogram (its A
//              entries are the identity).
// Jobs are cut into CTAs of kClCtaGroups 16-byte groups that never cross a job; each job carries its first CTA (a prefix sum), so what
// is planned and uploaded grows with jobs and steps, not with pixels.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/ifb200.h"

namespace ifb {

enum ClKind : uint32_t { kClTable = 0, kClMatrix = 1, kClWb = 2 };

// One segment of a job: `idx` is the table (kClTable / kClWb) or matrix (kClMatrix) index among the job's own.
struct ClSeg { uint32_t kind, idx; };

// One job.  px points at pixel (0, 0) of the window; `groups` 16-byte groups per row cover a row at any 4-byte phase.
// Its segments are segs[seg0, seg0 + nseg), its tables tables[tab0, tab0 + ntab) (1024 bytes each), its matrices mats[mat0, +nmat)
// (20 floats each).  wb_seg: the segment of its white balance (nseg when none) and wb its index among the call's white balances,
// whose 768 counters are hist[wb * 768, +768) (R, G, B) -- kClNone when none; low = the f64 area threshold.
struct ClJob {
    uint8_t* px;
    uint32_t w, h, stride, groups;
    uint32_t seg0, nseg, tab0, ntab, mat0, nmat, wb_seg, wb;
    double low;
};

constexpr uint32_t kClThreads = 256, kClCtaGroups = 2048, kClNone = 0xffffffffu;
constexpr uint32_t kClMaxSteps = IFB200_COLOR_MAX_STEPS;

struct ClWork {
    std::vector<ClJob> jobs;          // jobs that write pixels, in call order
    std::vector<uint32_t> first;      // first[i] = the first CTA of jobs[i]; first.back() = the number of CTAs of the apply launch
    std::vector<ClJob> wb_jobs;       // the jobs with a white balance, nseg cut to wb_seg (what the histogram evaluates), in order
    std::vector<uint32_t> wb_first;   // their prefix sum of CTAs (the histogram launch)
    std::vector<ClSeg> segs;
    std::vector<uint8_t> tables;      // 1024 bytes per table: [byte position 0..3][256]
    std::vector<float> mats;          // 20 floats per matrix
    // the last job planned without a white balance, whose segments, tables and matrices the next job shares when it has the same
    // steps array and format (the common case of many frames with one chain; a white balance's table is per job)
    const ifb200_color_step* last_steps = nullptr;
    uint32_t last_n = 0; int32_t last_am = -1;
    ClJob last{};
    uint64_t ctas() const { return first.empty() ? 0 : first.back(); }
    uint64_t wb_ctas() const { return wb_first.empty() ? 0 : wb_first.back(); }
    size_t bytes() const;             // what the plan uploads
};

// Empty when d is a valid descriptor, else why it is not; *code = the ifb200_status to fail with.
std::string color_check(const ifb200_color_desc& d, int* code);

// Appends the job of a valid descriptor (nothing for a job with no pixels or no steps).
void color_plan(const ifb200_color_desc& d, ClWork& wk);

// Checks every descriptor of one call, then plans all of them into wk.  Empty on success; else "color job i: <why>" for the first
// rejected descriptor, with *code = its status, and nothing planned.
std::string color_prepare(const ifb200_color_desc* d, size_t n, ClWork& wk, int* code);

// color.rs:101-108 uchar_clamp_ff on the host
uint8_t color_clamp(float v);

}  // namespace ifb
