// ifb_ycbcr.h -- host planner of ifb200_batch_ycbcr_to_bgra (include/ifb200.h: a JPEG's Y, Cb and Cr planes into BGRA, as libjpeg-turbo
// decodes into JCS_EXT_BGRA).  Product code, plain C++ without CUDA calls (tests/cpu_emu links it unchanged): validation of each
// descriptor, and one work item per job, in pixel_convert's plan shape (ifb_pixel_convert.h): 16-byte destination groups per row and
// a first-CTA prefix over the items, which each CTA of the one flat launch searches for its item.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/ifb200.h"
#include "ifb_pixel_convert.h"

namespace ifb {

// One work item: the whole w x h job.  A unit is destination group g of a row band: one row at 4:4:4 and 4:2:2, the two rows 2j and
// 2j + 1 that share chroma row j at 4:2:0 (one thread reads that chroma row and its halo once for both).  `groups` per destination row
// covers a row at any phase its stride allows; CTA c of the item takes the units [c * kYcCtaUnits, +kYcCtaUnits), band by band.
struct YcItem {
    const uint8_t* y; const uint8_t* cb; const uint8_t* cr; uint8_t* dst;
    uint32_t y_stride, cb_stride, cr_stride, dst_stride, w, h;
    uint32_t sampling, groups;
};

constexpr uint32_t kYcThreads = 256, kYcCtaUnits = 2048;

struct YcWork {
    std::vector<YcItem> items;
    std::vector<uint32_t> first;                   // first[i] = the first CTA of items[i]; first.back() = the number of CTAs
    uint64_t ctas() const { return first.empty() ? 0 : first.back(); }
};

// Rows and columns of a chroma plane of a w x h frame at `sampling` (0 x 0 for an unknown sampling).
uint32_t ycbcr_chroma_w(int32_t sampling, uint32_t w);
uint32_t ycbcr_chroma_h(int32_t sampling, uint32_t h);
// Row bands of an item: ceil(h / 2) at 4:2:0, else h.
uint32_t ycbcr_bands(uint32_t sampling, uint32_t h);

// The byte span [a, b) of a plane of `rows` (>= 1) rows of `row_bytes` bytes, `stride` apart; two planes overlap when their spans do.
struct Span { uintptr_t a, b; };
Span span_of(const uint8_t* p, uint32_t stride, uint32_t rows, uint64_t row_bytes);

// Empty when d is a valid descriptor, else why it is not; *code, when given, = IFB200_ERR_INVALID_ARGUMENT (its only status).
std::string ycbcr_check(const ifb200_ycbcr_desc& d, int* code = nullptr);

// Appends the work item of a valid descriptor (none for a job of zero area) and keeps wk.first a prefix sum with a trailing total.
void ycbcr_plan(const ifb200_ycbcr_desc& d, YcWork& wk);

// Checks every descriptor of one call, then plans all of them into wk.  Empty on success; else "ycbcr job i: <why>" for the first
// rejected descriptor, with *code = its status, and nothing planned.
std::string ycbcr_prepare(const ifb200_ycbcr_desc* d, size_t n, YcWork& wk, int* code);

}  // namespace ifb
