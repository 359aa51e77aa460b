// Executes imageflow_b200/csrc/ifb_watermark_kernel.cuh -- the product's CUDA source, unmodified, with the store epilogue it calls
// (ifb_finish.cuh, ifb_lut.cuh, ifb_types.cuh) -- on the CPU under a sequential emulation of the few CUDA built-ins it uses, with the
// product's host planner (ifb_watermark.cc, linked as it is).
// TEST INFRASTRUCTURE: nothing in the product calls it.  Neither kernel has a barrier or shared memory, so the threads of a CTA simply
// run one after the other.  Every canvas and F access of the composite goes through IFB_WM_LOAD* / IFB_WM_STORE*, which record the
// address of each 4-byte word they touch (a 16-byte pixel access records its four pixels; an F load records the pixel's first word)
// together with the CTA that made it.
#include "cuda_emu.h"

#include <cstddef>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/ifb200.h"
#include "../../imageflow_b200/csrc/ifb_watermark.h"

namespace emu {
static std::vector<uint64_t> loads, stores;            // (address, CTA) pairs, flattened
template <class T> static void rec(std::vector<uint64_t>& v, const T* p, size_t words) {
    for (size_t i = 0; i < words; ++i) { v.push_back((uint64_t)(uintptr_t)p + 4 * i); v.push_back(blockIdx.x); }
}
template <class T> static T load(const T* p) { rec(loads, p, sizeof(T) / 4); return *p; }
template <class T> static T loadf(const T* p) { rec(loads, p, 1); return *p; }
template <class T> static void store(T* p, const T& v) { rec(stores, p, sizeof(T) / 4); *p = v; }
}  // namespace emu
#define IFB_WM_LOAD4(p) emu::load(p)
#define IFB_WM_STORE4(p, v) emu::store(p, (uint32_t)(v))
#define IFB_WM_LOAD16(p) emu::load(p)
#define IFB_WM_STORE16(p, v) emu::store(p, (uint4)(v))
#define IFB_WM_LOADF(p) emu::loadf(p)

namespace ifbk {
#include "../../imageflow_b200/csrc/ifb_types.cuh"
#include "../../imageflow_b200/csrc/ifb_lut.cuh"
#include "../../imageflow_b200/csrc/ifb_finish.cuh"
#include "../../imageflow_b200/csrc/ifb_watermark_kernel.cuh"
}  // namespace ifbk

// The plan of a call, as ifb200_batch_watermark makes it: watermark_prepare, which watermark_locked (ifb_engine.cu) calls too.
// groups: 8 words per group (w, h, rows, tiles, job0, n, first, F byte offset); rep: the descriptor index of each group; opacity: what
// each group's copy gets (>= 1: none); jobs: 4 words per job (out address low, high, stride, groups).  Returns the CTAs of the composite, or -(ifb200_status) when a descriptor
// is rejected (err = why).
extern "C" long emu_watermark_plan(const ifb200_watermark_desc* d, size_t n, const float* t_lin, const float* t_srgb, uint32_t* groups,
                                   uint32_t* rep, float* opacity, size_t g_cap, uint32_t* jobs, size_t j_cap, size_t* n_groups,
                                   size_t* n_jobs, char* err, size_t err_cap) {
    ifb::WmWork wk;
    int code = 0;
    *n_groups = *n_jobs = 0;
    const std::string why = ifb::watermark_prepare(d, n, t_lin, t_srgb, wk, &code);
    if (!why.empty()) {
        snprintf(err, err_cap, "%s", why.c_str());
        return -code;
    }
    *n_groups = wk.groups.size(); *n_jobs = wk.jobs.size();
    for (size_t g = 0; g < wk.groups.size() && g < g_cap; ++g) {
        const ifb::WmGroup& q = wk.groups[g];
        const uint32_t v[8] = {q.w, q.h, q.rows, q.tiles, q.job0, q.n, q.first, (uint32_t)(uintptr_t)q.f};
        memcpy(groups + 8 * g, v, sizeof v);
        rep[g] = wk.rep[g]; opacity[g] = wk.opacity[g];
    }
    for (size_t j = 0; j < wk.jobs.size() && j < j_cap; ++j) {
        const uint64_t a = (uint64_t)(uintptr_t)wk.jobs[j].out;
        const uint32_t v[4] = {(uint32_t)a, (uint32_t)(a >> 32), wk.jobs[j].stride, wk.jobs[j].groups};
        memcpy(jobs + 4 * j, v, sizeof v);
    }
    return (long)wk.ctas();
}

// One call as the engine makes it, after the H pass: for each group g, vpass_f_kernel over inter[g] (its H-pass rows, in_h x w float4)
// with the V windows of axis[4 g .. 4 g + 3] (left, right, offsets, weights) into F + the group's offset, then ONE composite launch.
// in_h[g]: the source rows of group g.  tb: t_lin, t_srgb, lut16k.  loads / stores receive (address, CTA) pairs of the composite's pixel
// and F accesses (capacity cap pairs each).  sabotage != 0 corrupts the plan before the launches, to show that the checks of the tests
// catch it: 1 points the second group at the first group's F (a wrong F offset), 2 drops a 16-byte group from every row of the first
// job (rows cut short), 3 points the second job at the first job's rectangle (two jobs on one rectangle).
extern "C" long emu_watermark(const ifb200_watermark_desc* d, size_t n, const float* const* inter, const uint32_t* in_h,
                              const void* const* axis, float* F, const float* t_lin, const float* t_srgb, const uint8_t* lut16k,
                              uint64_t* loads, uint64_t* stores, size_t cap, size_t* n_loads, size_t* n_stores, char* err, size_t err_cap,
                              int sabotage) {
    ifb::WmWork wk;
    int code = 0;
    *n_loads = *n_stores = 0;
    const std::string why = ifb::watermark_prepare(d, n, t_lin, t_srgb, wk, &code);
    if (!why.empty()) {
        snprintf(err, err_cap, "%s", why.c_str());
        return -code;
    }
    for (auto& g : wk.groups) g.f = reinterpret_cast<const float*>(reinterpret_cast<uint8_t*>(F) + (uintptr_t)g.f);
    const ifbk::Tables tb{t_lin, t_srgb, lut16k};
    for (size_t g = 0; g < wk.groups.size(); ++g) {
        const ifb::WmGroup& q = wk.groups[g];
        const ifbk::AxisDev av{static_cast<const uint32_t*>(axis[4 * g]), static_cast<const uint32_t*>(axis[4 * g + 1]),
                               static_cast<const uint32_t*>(axis[4 * g + 2]), static_cast<const float*>(axis[4 * g + 3])};
        blockDim = {128, 1, 1};
        gridDim = {(q.w + 127) / 128, std::min<uint32_t>(q.h, 3u), 1};           // fewer rows of CTAs than rows: the y loop strides
        for (unsigned z = 0; z < 1; ++z)                                         // one group per launch here: blockIdx.z = 0
            for (unsigned by = 0; by < gridDim.y; ++by)
                for (unsigned bx = 0; bx < gridDim.x; ++bx)
                    for (unsigned t = 0; t < 128; ++t) {
                        blockIdx = {bx, by, z}; threadIdx = {t, 0, 0};
                        ifbk::vpass_f_kernel(av, in_h[g], q.w, q.h, reinterpret_cast<const float4*>(inter[g]),
                                             reinterpret_cast<float4*>(const_cast<float*>(q.f)));
                    }
    }
    if (sabotage == 1 && wk.groups.size() > 1) wk.groups[1].f = wk.groups[0].f;
    if (sabotage == 2 && !wk.jobs.empty()) wk.jobs[0].groups -= 1;
    if (sabotage == 3 && wk.jobs.size() > 1) { wk.jobs[1].out = wk.jobs[0].out; wk.jobs[1].stride = wk.jobs[0].stride; }
    emu::loads.clear(); emu::stores.clear();
    blockDim = {ifb::kWmThreads, 1, 1};
    gridDim = {(unsigned)wk.ctas(), 1, 1};
    for (unsigned b = 0; b < wk.ctas(); ++b)
        for (unsigned t = 0; t < ifb::kWmThreads; ++t) {
            blockIdx = {b, 0, 0}; threadIdx = {t, 0, 0};
            ifbk::watermark_composite_kernel(wk.groups.data(), (uint32_t)wk.groups.size(), wk.jobs.data(), tb, 0u);
        }
    *n_loads = emu::loads.size() / 2; *n_stores = emu::stores.size() / 2;
    for (size_t i = 0; i < emu::loads.size() && i < 2 * cap; ++i) loads[i] = emu::loads[i];
    for (size_t i = 0; i < emu::stores.size() && i < 2 * cap; ++i) stores[i] = emu::stores[i];
    return (long)wk.ctas();
}
