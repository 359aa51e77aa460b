// Executes imageflow_b200/csrc/ifb_canvas_kernel.cuh -- the product's CUDA source, unmodified -- on the CPU under a sequential
// emulation of the few CUDA built-ins it uses, with the product's host planner (ifb_canvas.cc, linked as it is).
// TEST INFRASTRUCTURE: nothing in the product calls it.  The kernel has no barrier and no shared memory, so the threads of a CTA
// simply run one after the other.  Every load and store goes through IFB_CV_LOAD* / IFB_CV_STORE*, which record the address of
// each 4-byte pixel they touch (a 16-byte access records its four pixels).
#include "cuda_emu.h"

#include <cstddef>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/ifb200.h"
#include "../../imageflow_b200/csrc/ifb_canvas.h"

namespace emu {
static std::vector<uint64_t> loads, stores;
template <class T> static void rec(std::vector<uint64_t>& v, const T* p) {
    for (size_t i = 0; i < sizeof(T) / 4; ++i) v.push_back((uint64_t)(uintptr_t)p + 4 * i);
}
template <class T> static T load(const T* p) { rec(loads, p); return *p; }
template <class T> static void store(T* p, const T& v) { rec(stores, p); *p = v; }
}  // namespace emu
#define IFB_CV_LOAD4(p) emu::load(p)
#define IFB_CV_STORE4(p, v) emu::store(p, (uint32_t)(v))
#define IFB_CV_LOAD16(p) emu::load(p)
#define IFB_CV_STORE16(p, v) emu::store(p, (uint4)(v))

namespace ifbk {
#include "../../imageflow_b200/csrc/ifb_canvas_kernel.cuh"
}  // namespace ifbk

// One call of ifb200_batch_canvas over d[0..n) as the engine makes it: canvas_prepare, which canvas_locked (ifb_engine.cu) calls
// too, then one launch.  loads / stores receive the address of every pixel access, in order (capacity cap each;
// *n_loads / *n_stores = the counts).  Returns the number of CTAs launched, or -1 when a descriptor is rejected (err = why).
// sabotage != 0 corrupts the plan before the launch, to show that the checks of the tests catch it: 1 runs the first tile twice,
// 2 moves the first item one pixel to the right, 3 drops the last tile.
extern "C" long emu_canvas(const ifb200_canvas_desc* d, size_t n, uint64_t* loads, uint64_t* stores, size_t cap, size_t* n_loads,
                           size_t* n_stores, char* err, size_t err_cap, int sabotage) {
    ifb::CvWork wk;
    int code = 0;
    const std::string why = ifb::canvas_prepare(d, n, wk, &code);
    if (!why.empty()) {
        snprintf(err, err_cap, "%s", why.c_str());
        return -1;
    }
    if (sabotage == 1 && !wk.tiles.empty()) wk.tiles.push_back(wk.tiles.front());
    if (sabotage == 2 && !wk.items.empty()) wk.items.front().dst += 4;
    if (sabotage == 3 && !wk.tiles.empty()) wk.tiles.pop_back();
    emu::loads.clear(); emu::stores.clear();
    for (unsigned b = 0; b < wk.tiles.size(); ++b) {
        emu::blockIdx = {b, 0, 0};
        for (unsigned t = 0; t < ifb::kCvThreads; ++t) {
            emu::threadIdx = {t, 0, 0};
            ifbk::canvas_kernel(wk.items.data(), wk.tiles.data());
        }
    }
    *n_loads = emu::loads.size(); *n_stores = emu::stores.size();
    for (size_t i = 0; i < emu::loads.size() && i < cap; ++i) loads[i] = emu::loads[i];
    for (size_t i = 0; i < emu::stores.size() && i < cap; ++i) stores[i] = emu::stores[i];
    return (long)wk.tiles.size();
}
