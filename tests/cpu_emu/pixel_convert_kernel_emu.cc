// Executes imageflow_b200/csrc/ifb_pixel_convert_kernel.cuh -- the product's CUDA source, unmodified -- on the CPU under a sequential
// emulation of the few CUDA built-ins it uses, with the product's host planner (ifb_pixel_convert.cc, linked as it is).
// TEST INFRASTRUCTURE: nothing in the product calls it.  The kernel has no barrier and no shared memory, so each CTA's threads simply
// run one after the other.  Every global load and store records the address of each byte it touches, with its width.
#include "cuda_emu.h"

#include <cstddef>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/ifb200.h"
#include "../../imageflow_b200/csrc/ifb_pixel_convert.h"

namespace emu {
static std::vector<uint64_t> loads, stores;      // (byte address << 8) | access width in bytes
template <class T> static void rec(std::vector<uint64_t>& v, const T* p) {
    for (size_t i = 0; i < sizeof(T); ++i) v.push_back(((uint64_t)(uintptr_t)p + i) << 8 | sizeof(T));
}
template <class T> static T load(const T* p) {
    rec(loads, p);
    return *p;
}
template <class T> static void store(T* p, const T& v) {
    rec(stores, p);
    *p = v;
}
}  // namespace emu
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t shift) {
    return (uint32_t)((((uint64_t)hi << 32) | lo) >> (shift & 31));
}
#define IFB_PC_LOAD1(p) emu::load(p)
#define IFB_PC_LOAD4(p) emu::load(p)
#define IFB_PC_STORE1(p, v) emu::store(p, (uint8_t)(v))
#define IFB_PC_STORE4(p, v) emu::store(p, (uint32_t)(v))
#define IFB_PC_STORE16(p, v) emu::store(p, (uint4)(v))

namespace ifbk {
#include "../../imageflow_b200/csrc/ifb_pixel_convert_kernel.cuh"
}  // namespace ifbk

// One call of ifb200_batch_pixel_convert over d[0..n) as the engine makes it: pixel_convert_prepare, which pixel_convert_locked
// (ifb_engine.cu) calls too, then one launch.  loads / stores receive (byte address << 8 | width) of every byte accessed, in order
// (capacity cap each; *n_loads / *n_stores = the counts).  Returns the number of CTAs launched, or -1 when a descriptor is rejected
// (err = why).  *n_items = the work items planned.
// sabotage != 0 corrupts the plan before the launch, to show that the checks of the tests catch it: 1 moves the second item's first
// CTA one later (the first item runs one CTA past its end, the second loses its first), 2 cuts the first item's rows short by one,
// 3 points the second item's destination at the first's (two jobs on one rectangle).
extern "C" long emu_pixel_convert(const ifb200_pixel_convert_desc* d, size_t n, uint64_t* loads, uint64_t* stores, size_t cap,
                                  size_t* n_loads, size_t* n_stores, size_t* n_items, char* err, size_t err_cap, int sabotage) {
    ifb::PcWork wk;
    int code = 0;
    const std::string why = ifb::pixel_convert_prepare(d, n, wk, &code);
    if (!why.empty()) {
        snprintf(err, err_cap, "%s", why.c_str());
        return -1;
    }
    *n_items = wk.items.size();
    if (sabotage == 1 && wk.items.size() > 1) wk.first[1] += 1;
    if (sabotage == 2 && !wk.items.empty()) wk.items.front().h -= 1;
    if (sabotage == 3 && wk.items.size() > 1) {
        wk.items[1].dst = wk.items[0].dst;
        wk.items[1].dst_stride = wk.items[0].dst_stride;
    }
    const uint64_t ctas = wk.ctas();
    emu::loads.clear(); emu::stores.clear();
    for (unsigned b = 0; b < ctas; ++b) {
        emu::blockIdx = {b, 0, 0};
        for (unsigned t = 0; t < ifb::kPcThreads; ++t) {
            emu::threadIdx = {t, 0, 0};
            ifbk::pixel_convert_kernel(wk.items.data(), wk.first.data(), (uint32_t)wk.items.size());
        }
    }
    *n_loads = emu::loads.size(); *n_stores = emu::stores.size();
    for (size_t i = 0; i < emu::loads.size() && i < cap; ++i) loads[i] = emu::loads[i];
    for (size_t i = 0; i < emu::stores.size() && i < cap; ++i) stores[i] = emu::stores[i];
    return (long)ctas;
}

// The plan alone: the number of work items and CTAs of one call (-1 when a descriptor is rejected).
extern "C" long emu_pixel_convert_plan(const ifb200_pixel_convert_desc* d, size_t n, size_t* n_items) {
    ifb::PcWork wk;
    int code = 0;
    if (!ifb::pixel_convert_prepare(d, n, wk, &code).empty()) return -1;
    *n_items = wk.items.size();
    return (long)wk.ctas();
}
