// Executes imageflow_b200/csrc/ifb_round_corners_kernel.cuh -- the product's CUDA source, unmodified -- on the CPU under a
// sequential emulation of the few CUDA built-ins it uses, with the product's host planner (ifb_round_corners.cc, linked as it is).
// TEST INFRASTRUCTURE: nothing in the product calls it.  The kernel has no barrier and no shared memory, so the threads of a CTA
// simply run one after the other.  Every pixel load and store goes through IFB_RC_LOAD / IFB_RC_STORE, which record the address.
#include <cmath>
#include <cstddef>
#include <cstdint>
#include <vector>

#include "../../include/ifb200.h"
#include "../../imageflow_b200/csrc/ifb_round_corners.h"

namespace emu {
struct Idx { unsigned x, y, z; };
static Idx threadIdx, blockIdx;
static std::vector<uint64_t> loads, stores;
}  // namespace emu
#define __global__
#define __device__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)
using emu::blockIdx;
using emu::threadIdx;
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline float __fsqrt_rn(float a) { return std::sqrt(a); }
static inline float __uint2float_rn(unsigned v) { return (float)v; }
#define IFB_RC_LOAD(p) (emu::loads.push_back((uint64_t)(uintptr_t)(p)), *(p))
#define IFB_RC_STORE(p, v) (emu::stores.push_back((uint64_t)(uintptr_t)(p)), *(p) = (v))

namespace ifbk {
#include "../../imageflow_b200/csrc/ifb_types.cuh"
#include "../../imageflow_b200/csrc/ifb_lut.cuh"
#include "../../imageflow_b200/csrc/ifb_round_corners_kernel.cuh"
}  // namespace ifbk

// One launch over descs[0..n) as ifb200_batch_round_corners makes it (ifb_engine.cu: round_corners_job, RcWork, round_corners_launch).
// loads / stores receive the byte address of every pixel access, in order (capacity cap each; *n_loads / *n_stores = the counts).
// Returns the number of CTAs launched, or -1 for a bad mode.
extern "C" long emu_round_corners(const ifb200_round_corners_desc* d, size_t n, const float* t_lin, const uint8_t* lut16k,
                                  uint64_t* loads, uint64_t* stores, size_t cap, size_t* n_loads, size_t* n_stores) {
    std::vector<ifb::RcJob> jobs;
    std::vector<ifb::RcTile> tiles;
    std::vector<ifb::RcRect> rects;
    for (size_t i = 0; i < n; ++i) {
        if (d[i].w == 0 || d[i].h == 0) continue;
        ifb::RcJob job{};
        if (!ifb::round_corners_plan(d[i].mode, d[i].radius, d[i].w, d[i].h, &job)) return -1;
        job.px = d[i].px; job.stride = d[i].stride;
        job.matte = (uint32_t)d[i].matte_bgra[0] | ((uint32_t)d[i].matte_bgra[1] << 8) | ((uint32_t)d[i].matte_bgra[2] << 16) |
                    ((uint32_t)d[i].matte_bgra[3] << 24);
        rects.clear();
        ifb::round_corners_cover(job, rects);
        const uint32_t j = (uint32_t)jobs.size();
        jobs.push_back(job);
        for (const auto& r : rects) {
            const uint64_t area = (uint64_t)r.w * r.h;
            for (uint64_t f = 0; f < area; f += ifb::kRcTilePixels)
                tiles.push_back({j, r.x0, r.y0, r.w, (uint32_t)f, (uint32_t)(area - f < ifb::kRcTilePixels ? area - f : ifb::kRcTilePixels)});
        }
    }
    emu::loads.clear(); emu::stores.clear();
    const ifbk::Tables tb{t_lin, nullptr, lut16k};
    for (unsigned b = 0; b < tiles.size(); ++b) {
        emu::blockIdx = {b, 0, 0};
        for (unsigned t = 0; t < ifb::kRcThreads; ++t) {
            emu::threadIdx = {t, 0, 0};
            ifbk::round_corners_kernel(jobs.data(), tiles.data(), tb);
        }
    }
    *n_loads = emu::loads.size(); *n_stores = emu::stores.size();
    for (size_t i = 0; i < emu::loads.size() && i < cap; ++i) loads[i] = emu::loads[i];
    for (size_t i = 0; i < emu::stores.size() && i < cap; ++i) stores[i] = emu::stores[i];
    return (long)tiles.size();
}
