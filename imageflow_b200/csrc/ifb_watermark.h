// ifb_watermark.h -- host planner of ifb200_batch_watermark (include/ifb200.h: watermark composites that share one resample per distinct
// watermark image).  Product code, plain C++ without CUDA calls (tests/cpu_emu links it unchanged): validation of each descriptor, the
// grouping of jobs by F (the resampled premultiplied working-space watermark, which depends only on the watermark's bytes, format, applied
// opacity, target size, filter, sharpen and working space), and the composite launch cut into CTAs.
//
// Composite CTA order: group by group; inside a group, F tile by F tile; inside a tile, job by job.  So consecutive CTAs read the same
// F tile for different frames, and F is served from L2 after its first read.  Each group carries its first CTA (a prefix sum), so what
// is planned and uploaded grows with jobs and groups, not with pixels.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/ifb200.h"

namespace ifb {

// One composite: the frame's rectangle (origin at (x, y) of the canvas), its stride, the 16-byte groups per row that cover a row of w
// pixels at any 4-byte phase, the store flags (JobDev's: linear, alpha, compose) and the premultiplied matte (BlendWithMatte only).
struct WmJob {
    uint8_t* out;
    uint32_t stride, groups, flags, pad_;
    float matte[4];
};

// One F: w x h float4 pixels at f (row pitch w), shared by jobs [job0, job0 + n) of WmWork::jobs.  Tiles of `rows` rows; the group's
// CTAs are [first, first + tiles * n).
struct WmGroup {
    const float* f;
    uint32_t w, h, rows, tiles, job0, n, first, pad_;
};

constexpr uint32_t kWmThreads = 256, kWmTilePixels = 4096;

struct WmWork {
    std::vector<WmGroup> groups;      // f is the byte offset of the group's F in the call's F buffer until the engine rebases it
    std::vector<WmJob> jobs;          // grouped: the jobs of groups[g] are jobs[groups[g].job0, + n)
    std::vector<uint32_t> rep;        // rep[g]: a descriptor index of group g (its draw is the resample of F)
    std::vector<float> opacity;       // opacity[g]: the opacity applied to group g's copy, or a value >= 1 for none
    uint64_t f_bytes = 0;             // the F buffer
    uint64_t ctas() const { return groups.empty() ? 0 : (uint64_t)groups.back().first + (uint64_t)groups.back().tiles * groups.back().n; }
    size_t bytes() const { return groups.size() * sizeof(WmGroup) + jobs.size() * sizeof(WmJob); }   // what the plan uploads
};

// The argument checks of one scale_and_render job (scaling.rs:24-48), as ifb200_batch_enqueue makes them: empty when valid, else why
// not; *code = the ifb200_status to fail with.
std::string resample_check(const ifb200_resample_desc& d, int* code);

// Empty when d is a valid descriptor (or a skipped zero-area job), else why it is not; *code = the ifb200_status to fail with.
std::string watermark_check(const ifb200_watermark_desc& d, int* code);

// watermark.rs:166: opacity.clamp(0, 1), and whether it is applied (< 1; NaN is not)
bool watermark_opacity(float opacity, float* applied);

// Plans d[0..n) (all checked): groups, jobs and CTAs.  t_lin / t_srgb: byte_to_float tables (for the matte, as make_job).
void watermark_plan(const ifb200_watermark_desc* d, size_t n, const float* t_lin, const float* t_srgb, WmWork& wk);

// Checks every descriptor of one call, then plans all of them into wk.  Empty on success; else "watermark job i: <why>" for the first
// rejected descriptor, with *code = its status, and nothing planned.
std::string watermark_prepare(const ifb200_watermark_desc* d, size_t n, const float* t_lin, const float* t_srgb, WmWork& wk, int* code);

}  // namespace ifb
