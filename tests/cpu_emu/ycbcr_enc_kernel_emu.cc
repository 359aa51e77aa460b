// Executes imageflow_b200/csrc/ifb_ycbcr_enc_kernel.cuh -- the product's CUDA source, unmodified, with the matte helpers
// (ifb_matte.cuh, ifb_lut.cuh, ifb_types.cuh) and pixel_convert's item search it uses -- on the CPU under a sequential emulation of the
// few CUDA built-ins they use, with the product's host planner (ifb_ycbcr_enc.cc, ifb_ycbcr.cc and ifb_pixel_convert.cc, linked as
// they are).
// TEST INFRASTRUCTURE: nothing in the product calls it.  The kernel has no barrier and no shared memory, so each CTA's threads simply
// run one after the other.  Every global load and store of the kernel records the address of each byte it touches, with its width;
// every sample is asserted to lie in 0..255 before it is stored.
#include "cuda_emu.h"

#include <cassert>
#include <cstddef>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/ifb200.h"
#include "../../imageflow_b200/csrc/ifb_ycbcr_enc.h"

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
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t shift) {      // for pixel_convert's own kernel, which
    return (uint32_t)((((uint64_t)hi << 32) | lo) >> (shift & 31));                       // the included header also defines
}
#define IFB_PC_LOAD1(p) emu::load(p)
#define IFB_PC_LOAD4(p) emu::load(p)
#define IFB_PC_STORE1(p, v) emu::store(p, (uint8_t)(v))
#define IFB_PC_STORE4(p, v) emu::store(p, (uint32_t)(v))
#define IFB_PC_STORE16(p, v) emu::store(p, (uint4)(v))
#define IFB_YE_LOAD4(p) emu::load(p)
#define IFB_YE_LOAD16(p) emu::load(p)
#define IFB_YE_STORE1(p, v) emu::store(p, (uint8_t)(v))
#define IFB_YE_STORE4(p, v) emu::store(p, (uint32_t)(v))
#define IFB_YE_STORE8(p, v) emu::store(p, (unsigned long long)(v))
#define IFB_YE_ASSERT(c) assert(c)

namespace ifbk {
#include "../../imageflow_b200/csrc/ifb_types.cuh"
#include "../../imageflow_b200/csrc/ifb_lut.cuh"
#include "../../imageflow_b200/csrc/ifb_matte.cuh"
#include "../../imageflow_b200/csrc/ifb_pixel_convert_kernel.cuh"
#include "../../imageflow_b200/csrc/ifb_ycbcr_enc_kernel.cuh"
}  // namespace ifbk

// One call of ifb200_batch_bgra_to_ycbcr over d[0..n) as the engine makes it: bgra_to_ycbcr_prepare, which bgra_to_ycbcr_locked
// (ifb_engine.cu) calls too, then one launch with the library's tables t_lin and lut16k.  loads / stores receive (byte address << 8 |
// width) of every byte accessed, in order (capacity cap each; *n_loads / *n_stores = the counts).  Returns the number of CTAs launched,
// or -1 when a descriptor is rejected (err = why).  *n_items = the work items planned.
// sabotage != 0 corrupts the plan before the launch, to show that the checks of the tests catch it: 1 moves the second item's first
// CTA one later, 2 cuts the first item's rows short by one, 3 points the second item's Cb plane at its Cr plane, 4 drops the first
// item's matte flag.
extern "C" long emu_bgra_to_ycbcr(const ifb200_bgra_to_ycbcr_desc* d, size_t n, const float* t_lin, const uint8_t* lut16k,
                                  uint64_t* loads, uint64_t* stores, size_t cap, size_t* n_loads, size_t* n_stores, size_t* n_items,
                                  char* err, size_t err_cap, int sabotage) {
    ifb::YeWork wk;
    int code = 0;
    const std::string why = ifb::bgra_to_ycbcr_prepare(d, n, wk, &code);
    if (!why.empty()) {
        snprintf(err, err_cap, "%s", why.c_str());
        return -1;
    }
    *n_items = wk.items.size();
    if (sabotage == 1 && wk.items.size() > 1) wk.first[1] += 1;
    if (sabotage == 2 && !wk.items.empty()) wk.items.front().h -= 1;
    if (sabotage == 3 && wk.items.size() > 1) {
        wk.items[1].cb = wk.items[1].cr;
        wk.items[1].cb_stride = wk.items[1].cr_stride;
    }
    if (sabotage == 4 && !wk.items.empty()) wk.items.front().alpha = 0;
    const ifbk::Tables tb{t_lin, nullptr, lut16k};
    const uint64_t ctas = wk.ctas();
    emu::loads.clear(); emu::stores.clear();
    for (unsigned b = 0; b < ctas; ++b) {
        emu::blockIdx = {b, 0, 0};
        for (unsigned t = 0; t < ifb::kYeThreads; ++t) {
            emu::threadIdx = {t, 0, 0};
            ifbk::bgra_to_ycbcr_kernel(wk.items.data(), wk.first.data(), (uint32_t)wk.items.size(), tb);
        }
    }
    *n_loads = emu::loads.size(); *n_stores = emu::stores.size();
    for (size_t i = 0; i < emu::loads.size() && i < cap; ++i) loads[i] = emu::loads[i];
    for (size_t i = 0; i < emu::stores.size() && i < cap; ++i) stores[i] = emu::stores[i];
    return (long)ctas;
}

// The plan alone: the number of work items and CTAs of one call (-1 when a descriptor is rejected), and each item's first CTA.
extern "C" long emu_bgra_to_ycbcr_plan(const ifb200_bgra_to_ycbcr_desc* d, size_t n, size_t* n_items, uint32_t* first, size_t first_cap) {
    ifb::YeWork wk;
    int code = 0;
    if (!ifb::bgra_to_ycbcr_prepare(d, n, wk, &code).empty()) return -1;
    *n_items = wk.items.size();
    for (size_t i = 0; i < wk.first.size() && i < first_cap; ++i) first[i] = wk.first[i];
    return (long)wk.ctas();
}
