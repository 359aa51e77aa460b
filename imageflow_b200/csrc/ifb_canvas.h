// ifb_canvas.h -- host planner of the canvas operations of ifb200_batch_canvas (include/ifb200.h: fill_rectangle, copy_rectangle,
// ExpandCanvas, normalize_unused_alpha).  Product code, plain C++ without CUDA calls (tests/cpu_emu links it unchanged): validation of
// each descriptor, and the cut of every job into disjoint rectangle work items, which are cut into CTA tiles of one flat launch.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/ifb200.h"

namespace ifb {

// What a work item does to each pixel of its rectangle.
enum CvKind : uint32_t {
    kCvFill = 0,                                   // dst = color
    kCvCopy = 1,                                   // dst = src (| 0xFF000000 with kCvOrAlpha; then also src = that with kCvWriteBack)
    kCvOpaque = 2,                                 // dst |= 0xFF000000, in place
};
enum : uint32_t { kCvOrAlpha = 1, kCvWriteBack = 2 };

// One rectangle of w x h pixels.  dst / src point at its top-left pixel.  The kernel walks each row in 16-byte groups aligned to
// dst's addresses: `groups` per row covers a row at any of the four 4-byte phases a row of dst can have.
struct CvItem {
    uint8_t* dst; uint8_t* src;
    uint32_t dst_stride, src_stride, w, h, groups;
    uint32_t kind, flags, color;                   // color: BGRA8 packed little-endian (b | g << 8 | r << 16 | a << 24)
};

// One CTA of canvas_kernel: groups [first, first + count) of item `item`, counted row by row (row = k / groups, group = k % groups).
constexpr uint32_t kCvThreads = 256, kCvTileGroups = 4096;
struct CvTile { uint32_t item, first, count; };

struct CvWork {
    std::vector<CvItem> items; std::vector<CvTile> tiles;
};

// Empty when d is a valid descriptor, else why it is not; *code, when given, = IFB200_ERR_INVALID_ARGUMENT (its only status).
std::string canvas_check(const ifb200_canvas_desc& d, int* code = nullptr);

// Appends the work items of a valid descriptor and their tiles to `wk`: disjoint rectangles, so that every pixel the op writes is
// written by one thread, once.  Nothing for a job that writes no pixel.
void canvas_plan(const ifb200_canvas_desc& d, CvWork& wk);

// Checks every descriptor of one call, then plans all of them into wk.  Empty on success; else "canvas job i: <why>" for the first
// rejected descriptor, with *code = its status, and nothing planned.
std::string canvas_prepare(const ifb200_canvas_desc* d, size_t n, CvWork& wk, int* code);

}  // namespace ifb
