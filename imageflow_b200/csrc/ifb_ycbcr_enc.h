// ifb_ycbcr_enc.h -- host planner of ifb200_batch_bgra_to_ycbcr (include/ifb200.h: BGRA frames into a JPEG encoder's Y, Cb and Cr
// planes, as libjpeg-turbo's compressor forms them from JCS_EXT_BGRA).  Product code, plain C++ without CUDA calls (tests/cpu_emu
// links it unchanged): validation of each descriptor, and one work item per job, in pixel_convert's plan shape (ifb_pixel_convert.h):
// units per row and a first-CTA prefix over the items, which each CTA of the one flat launch searches for its item.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/ifb200.h"
#include "ifb_pixel_convert.h"

namespace ifb {

// One work item: the whole w x h job.  A unit is a run of kYeRun source columns [kYeRun u, +kYeRun) of a row band: one row at 4:4:4
// and 4:2:2, the row pair 2j and 2j + 1 that makes chroma row j at 4:2:0 (one thread holds both rows of every box it sums).  Runs
// start at even columns, so no chroma sample takes pixels of two units.  CTA c of the item takes the units
// [c * kYeCtaUnits, +kYeCtaUnits), band by band.  matte is the descriptor's matte_bgra as a little-endian word.
struct YeItem {
    const uint8_t* src; uint8_t* y; uint8_t* cb; uint8_t* cr;
    uint32_t src_stride, y_stride, cb_stride, cr_stride, w, h;
    uint32_t sampling, units, alpha, matte;
};

constexpr uint32_t kYeThreads = 256, kYeCtaUnits = 1024, kYeRun = 8;

struct YeWork {
    std::vector<YeItem> items;
    std::vector<uint32_t> first;                   // first[i] = the first CTA of items[i]; first.back() = the number of CTAs
    uint64_t ctas() const { return first.empty() ? 0 : first.back(); }
};

// Empty when d is a valid descriptor, else why it is not; *code, when given, = IFB200_ERR_INVALID_ARGUMENT (its only status).
std::string bgra_to_ycbcr_check(const ifb200_bgra_to_ycbcr_desc& d, int* code = nullptr);

// Appends the work item of a valid descriptor (none for a job of zero area) and keeps wk.first a prefix sum with a trailing total.
void bgra_to_ycbcr_plan(const ifb200_bgra_to_ycbcr_desc& d, YeWork& wk);

// Checks every descriptor of one call, then plans all of them into wk.  Empty on success; else "bgra_to_ycbcr job i: <why>" for the
// first rejected descriptor, with *code = its status, and nothing planned.
std::string bgra_to_ycbcr_prepare(const ifb200_bgra_to_ycbcr_desc* d, size_t n, YeWork& wk, int* code);

}  // namespace ifb
