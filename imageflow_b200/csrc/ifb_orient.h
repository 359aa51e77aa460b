// ifb_orient.h -- host planner of ifb200_batch_orient (include/ifb200.h: the eight EXIF orientations as one gather).  Product code,
// plain C++ without CUDA calls (tests/cpu_emu links it unchanged): validation of each descriptor, and at most two work items per job.
// Items carry their first CTA (a prefix sum of per-item CTA counts), so what is planned and uploaded grows with the number of jobs,
// not with pixels; each CTA of the one flat launch finds its item by a binary search over that prefix.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/ifb200.h"

namespace ifb {

enum OrKind : uint32_t {
    kOrTile = 0,                                   // 5..8: tiles through shared memory
    kOrRow = 1,                                    // 1..4 out of place: output rows gathered in 16-byte groups
    kOrPair = 2,                                   // 2..4 in place: each thread swaps a group of pixels with its mirror image
};
// kOrFx: the source x is reversed (w-1-x for rows and pairs, w-1-y for tiles); kOrFy: the source y is (h-1-y, or h-1-x for tiles)
enum : uint32_t { kOrFx = 1, kOrFy = 2 };

// One work item.  in / out point at pixel (0, 0) of the job's windows (out == in for kOrPair); w x h is the INPUT window.
//   kOrTile: tiles of 32 source columns x kOrTileOx output columns; `groups` = tiles across the source width.  CTA c of the item
//            takes the source columns [32 (c % groups), +32) and the output columns [kOrTileOx (c / groups), +kOrTileOx).
//   kOrRow / kOrPair: the rows [y0, y0 + rows) of the output (kOrRow) or of the pair domain (kOrPair), pixels [0, xlim) of each,
//            walked in 16-byte groups aligned to the addresses of those rows; `groups` per row covers a row at any of the four
//            4-byte phases.  CTA c takes the groups [c * kOrCtaGroups, +kOrCtaGroups), counted row by row.
struct OrItem {
    const uint8_t* in; uint8_t* out;
    uint32_t in_stride, out_stride, w, h;
    uint32_t kind, flags, y0, rows, xlim, groups;
};

constexpr uint32_t kOrThreads = 256, kOrCtaGroups = 4096, kOrTileOx = 128;

struct OrWork {
    std::vector<OrItem> items;
    std::vector<uint32_t> first;                   // first[i] = the first CTA of items[i]; first.back() = the number of CTAs
    uint64_t ctas() const { return first.empty() ? 0 : first.back(); }
};

// 16-byte groups per row of xlim pixels starting at `row0`, for rows `stride` bytes apart: enough to cover every row whatever its
// 4-byte phase modulo 16 (also used by the colour planner, ifb_color.cc).
uint32_t groups_per_row(const uint8_t* row0, uint32_t stride, uint32_t xlim);

// The orientation a flag stands for: 2..8 as they are, every other value 1 (the identity).
int32_t orient_flag(int32_t orientation);

// Empty when d is a valid descriptor, else why it is not; *code, when given, = IFB200_ERR_INVALID_ARGUMENT (its only status).
std::string orient_check(const ifb200_orient_desc& d, int* code = nullptr);

// Appends the work items of a valid descriptor (none for a job that writes no pixel) and keeps wk.first a prefix sum with a
// trailing total.
void orient_plan(const ifb200_orient_desc& d, OrWork& wk);

// Checks every descriptor of one call, then plans all of them into wk.  Empty on success; else "orient job i: <why>" for the first
// rejected descriptor, with *code = its status, and nothing planned.
std::string orient_prepare(const ifb200_orient_desc* d, size_t n, OrWork& wk, int* code);

}  // namespace ifb
