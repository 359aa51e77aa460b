// ifb_profile.h -- host planner of ifb200_batch_transform_to_srgb and ifb200_source_profile_plan (include/ifb200.h: a decoder's colour
// profile to sRGB).  Product code, plain C++ without CUDA calls (tests/cpu_emu links it unchanged): the ICC parser (header, tag table,
// 'XYZ ', 'curv', 'para' and the refusals), the colorimetry of gAMA+cHRM and CICP (H.273 primaries, SDR transfer functions), the
// float64 tabulation and matrix, the sharing of one plan between identical profiles of a call, and one work item per job.  The items
// are pixel_convert's (ifb_pixel_convert.h: same row rules, same 16-byte destination groups, same first CTAs), each with the index of
// its plan.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/ifb200.h"
#include "ifb_pixel_convert.h"

namespace ifb {

constexpr uint32_t kPfBgra = 0x80000000u;           // PfWork::plan_of: the source is BGRA (no swizzle), else pixel_convert's op

struct PfWork {
    PcWork pc;                                      // the items and their first CTAs
    std::vector<uint32_t> plan_of;                  // per item: its index into plans, | kPfBgra for a BGRA source
    std::vector<ifb200_profile_plan> plans;         // the distinct profiles of the call, each planned once
};

// IFB200_OK and *plan filled, or IFB200_ERR_NOT_IMPLEMENTED / IFB200_ERR_INVALID_ARGUMENT with *why.
int profile_plan(const ifb200_source_profile& p, ifb200_profile_plan* plan, std::string* why);

// The plans of one call's profiles: identical profiles (compared byte for byte) share one plan, planned once.  Used by
// ifb200_batch_transform_to_srgb and ifb200_batch_enqueue_profiled.
struct ProfilePlans {
    std::vector<ifb200_profile_plan> plans;
    std::vector<const ifb200_source_profile*> planned;   // the profile each plan was made from
    // *index = the plan of p, planned now if no identical profile has been.  IFB200_OK, or the planner's status with *why.
    int add(const ifb200_source_profile& p, uint32_t* index, std::string* why);
};

// Checks every descriptor of one call and plans every distinct profile, then plans the items into wk.  Empty on success; else
// "transform to srgb job i: <why>" for the first rejected job, with *code = its status, and nothing planned.
std::string transform_to_srgb_prepare(const ifb200_to_srgb_desc* d, size_t n, PfWork& wk, int* code);

}  // namespace ifb
