// ifb_pixel_convert.h -- host planner of ifb200_batch_pixel_convert (include/ifb200.h: RGB24, RGBA, Gray8 and GrayAlpha8 rows into
// BGRA, and BGRA into RGB24).  Product code, plain C++ without CUDA calls (tests/cpu_emu links it unchanged): validation of each
// descriptor, and one work item per job.  Items carry their first CTA (a prefix sum of per-item CTA counts), so what is planned and
// uploaded grows with the number of jobs, not with pixels; each CTA of the one flat launch finds its item by a binary search over that
// prefix.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/ifb200.h"

namespace ifb {

// One work item: the whole w x h job.  Its destination rows are walked in 16-byte groups aligned to the destination's addresses;
// `groups` per row covers a row at any phase its stride allows.  CTA c of the item takes the groups [c * kPcCtaGroups, +kPcCtaGroups),
// counted row by row.
struct PcItem {
    const uint8_t* src; uint8_t* dst;
    uint32_t src_stride, dst_stride, w, h;
    uint32_t op, opaque, groups;
};

constexpr uint32_t kPcThreads = 256, kPcCtaGroups = 4096;

struct PcWork {
    std::vector<PcItem> items;
    std::vector<uint32_t> first;                   // first[i] = the first CTA of items[i]; first.back() = the number of CTAs
    uint64_t ctas() const { return first.empty() ? 0 : first.back(); }
};

// Bytes per pixel of op's source and destination (0 for an unknown op).
uint32_t pixel_src_bytes(int32_t op);
uint32_t pixel_dst_bytes(int32_t op);

// Empty when d is a valid descriptor, else why it is not; *code, when given, = IFB200_ERR_INVALID_ARGUMENT (its only status).
std::string pixel_convert_check(const ifb200_pixel_convert_desc& d, int* code = nullptr);

// Appends the work item of a valid descriptor (none for a job of zero area) and keeps wk.first a prefix sum with a trailing total.
void pixel_convert_plan(const ifb200_pixel_convert_desc& d, PcWork& wk);

// Checks every descriptor of one call, then plans all of them into wk.  Empty on success; else "pixel convert job i: <why>" for the
// first rejected descriptor, with *code = its status, and nothing planned.
std::string pixel_convert_prepare(const ifb200_pixel_convert_desc* d, size_t n, PcWork& wk, int* code);

}  // namespace ifb
