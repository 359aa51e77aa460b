// Executes imageflow_b200/csrc/ifb_profile_kernel.cuh -- the product's CUDA source, unmodified, with the pixel_convert and lut_encode
// device functions it calls -- on the CPU under a sequential emulation of the CUDA built-ins it uses, with the product's host planner
// (ifb_profile.cc, ifb_pixel_convert.cc and ifb_weights.cc, linked as they are).
// TEST INFRASTRUCTURE: nothing in the product calls it.  The kernel's one barrier is emulated by running every CTA twice: in pass 0
// every thread stages its share of the plan and returns at __syncthreads(); in pass 1 every thread stages again (the same values) and
// goes on past it.  Global pixel loads and stores of pass 1 record the address of each byte they touch, with the access width.
#include "cuda_emu.h"

#include <cstddef>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/ifb200.h"
#include "../../imageflow_b200/csrc/ifb_profile.h"

namespace emu {
static int pass, seg;
static std::vector<uint64_t> loads, stores;      // (byte address << 8) | access width in bytes
template <class T> static void rec(std::vector<uint64_t>& v, const T* p) {
    for (size_t i = 0; i < sizeof(T); ++i) v.push_back(((uint64_t)(uintptr_t)p + i) << 8 | sizeof(T));
}
template <class T> static T load(const T* p) {
    if (seg == pass) rec(loads, p);
    return *p;
}
template <class T> static void store(T* p, const T& v) {
    if (seg != pass) return;
    rec(stores, p);
    *p = v;
}
}  // namespace emu
static inline uint32_t __funnelshift_r(uint32_t lo, uint32_t hi, uint32_t shift) {
    return (uint32_t)((((uint64_t)hi << 32) | lo) >> (shift & 31));
}
#define __shared__ static
#define __syncthreads() do { if (emu::seg == emu::pass) return; ++emu::seg; } while (0)
#define IFB_PC_LOAD1(p) emu::load(p)
#define IFB_PC_LOAD4(p) emu::load(p)
#define IFB_PC_STORE1(p, v) emu::store(p, (uint8_t)(v))
#define IFB_PC_STORE4(p, v) emu::store(p, (uint32_t)(v))
#define IFB_PC_STORE16(p, v) emu::store(p, (uint4)(v))

namespace ifbk {
#include "../../imageflow_b200/csrc/ifb_lut.cuh"
#include "../../imageflow_b200/csrc/ifb_pixel_convert_kernel.cuh"
#include "../../imageflow_b200/csrc/ifb_profile_kernel.cuh"
}  // namespace ifbk

// One call of ifb200_batch_transform_to_srgb over d[0..n) as the engine makes it: transform_to_srgb_prepare, which
// transform_to_srgb_locked (ifb_engine.cu) calls too, then one launch.  loads / stores receive (byte address << 8 | width) of every
// byte accessed, in order (capacity cap each; *n_loads / *n_stores = the counts).  Returns the number of CTAs launched, or -(status)
// when a job is rejected (err = why).  *n_items = the work items planned, *n_plans = the profiles planned.
extern "C" long emu_transform_to_srgb(const ifb200_to_srgb_desc* d, size_t n, const uint8_t* lut16k, uint64_t* loads, uint64_t* stores,
                                      size_t cap, size_t* n_loads, size_t* n_stores, size_t* n_items, size_t* n_plans, char* err,
                                      size_t err_cap) {
    ifb::PfWork wk;
    int code = 0;
    const std::string why = ifb::transform_to_srgb_prepare(d, n, wk, &code);
    if (!why.empty()) {
        snprintf(err, err_cap, "%s", why.c_str());
        return -code;
    }
    *n_items = wk.pc.items.size();
    *n_plans = wk.plans.size();
    const uint64_t ctas = wk.pc.ctas();
    emu::loads.clear(); emu::stores.clear();
    for (unsigned b = 0; b < ctas; ++b) {
        emu::blockIdx = {b, 0, 0};
        for (emu::pass = 0; emu::pass < 2; ++emu::pass)
            for (unsigned t = 0; t < ifb::kPcThreads; ++t) {
                emu::threadIdx = {t, 0, 0};
                emu::seg = 0;
                ifbk::transform_to_srgb_kernel(wk.pc.items.data(), wk.pc.first.data(), wk.plan_of.data(), wk.plans.data(), lut16k,
                                               (uint32_t)wk.pc.items.size());
            }
    }
    *n_loads = emu::loads.size(); *n_stores = emu::stores.size();
    for (size_t i = 0; i < emu::loads.size() && i < cap; ++i) loads[i] = emu::loads[i];
    for (size_t i = 0; i < emu::stores.size() && i < cap; ++i) stores[i] = emu::stores[i];
    return (long)ctas;
}

// The planner alone on a copy of the profile's bytes in a buffer of exactly icc_len bytes (so that AddressSanitizer sees any read
// past its end): the status of ifb200_source_profile_plan, with why.
extern "C" int emu_profile_plan(const ifb200_source_profile* p, char* why, size_t why_cap) {
    ifb200_source_profile q = *p;
    std::vector<uint8_t> bytes(p->icc, p->icc + (p->icc ? p->icc_len : 0));
    uint8_t* exact = bytes.empty() ? nullptr : new uint8_t[bytes.size()];
    if (exact) std::memcpy(exact, bytes.data(), bytes.size());
    if (exact) q.icc = exact;
    ifb200_profile_plan plan;
    std::string reason;
    const int code = ifb::profile_plan(q, &plan, &reason);
    delete[] exact;
    snprintf(why, why_cap, "%s", reason.c_str());
    return code;
}
