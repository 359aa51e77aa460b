// Executes imageflow_b200/csrc/ifb_round_corners_kernel.cuh -- the product's CUDA source, unmodified -- on the CPU under a
// sequential emulation of the few CUDA built-ins it uses, with the product's host planner (ifb_round_corners.cc, linked as it is).
// TEST INFRASTRUCTURE: nothing in the product calls it.  The kernel has no barrier and no shared memory, so the threads of a CTA
// simply run one after the other.  Every pixel load and store goes through IFB_RC_LOAD / IFB_RC_STORE, which record the address.
#include "cuda_emu.h"

#include <cstddef>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/ifb200.h"
#include "../../imageflow_b200/csrc/ifb_round_corners.h"

namespace emu {
static std::vector<uint64_t> loads, stores;
}  // namespace emu
#define IFB_RC_LOAD(p) (emu::loads.push_back((uint64_t)(uintptr_t)(p)), *(p))
#define IFB_RC_STORE(p, v) (emu::stores.push_back((uint64_t)(uintptr_t)(p)), *(p) = (v))

namespace ifbk {
#include "../../imageflow_b200/csrc/ifb_types.cuh"
#include "../../imageflow_b200/csrc/ifb_lut.cuh"
#include "../../imageflow_b200/csrc/ifb_round_corners_kernel.cuh"
}  // namespace ifbk

// One call of ifb200_batch_round_corners over d[0..n) as the engine makes it: round_corners_prepare, which round_corners_locked
// (ifb_engine.cu) calls too, then one launch.  loads / stores receive the byte address of every pixel access, in order (capacity
// cap each; *n_loads / *n_stores = the counts).  Returns the number of CTAs launched, or -1 when a descriptor is rejected (err = why).
extern "C" long emu_round_corners(const ifb200_round_corners_desc* d, size_t n, const float* t_lin, const uint8_t* lut16k,
                                  uint64_t* loads, uint64_t* stores, size_t cap, size_t* n_loads, size_t* n_stores, char* err, size_t err_cap) {
    ifb::RcWork wk;
    int code = 0;
    const std::string why = ifb::round_corners_prepare(d, n, wk, &code);
    if (!why.empty()) {
        snprintf(err, err_cap, "%s", why.c_str());
        return -1;
    }
    emu::loads.clear(); emu::stores.clear();
    const ifbk::Tables tb{t_lin, nullptr, lut16k};
    for (unsigned b = 0; b < wk.tiles.size(); ++b) {
        emu::blockIdx = {b, 0, 0};
        for (unsigned t = 0; t < ifb::kRcThreads; ++t) {
            emu::threadIdx = {t, 0, 0};
            ifbk::round_corners_kernel(wk.jobs.data(), wk.tiles.data(), tb);
        }
    }
    *n_loads = emu::loads.size(); *n_stores = emu::stores.size();
    for (size_t i = 0; i < emu::loads.size() && i < cap; ++i) loads[i] = emu::loads[i];
    for (size_t i = 0; i < emu::stores.size() && i < cap; ++i) stores[i] = emu::stores[i];
    return (long)wk.tiles.size();
}
