// Executes imageflow_b200/csrc/ifb_color_kernel.cuh -- the product's CUDA source, unmodified -- on the CPU under a sequential
// emulation of the few CUDA built-ins it uses, with the product's host planner (ifb_color.cc, linked as it is).
// TEST INFRASTRUCTURE: nothing in the product calls it.  Barriers are emulated by running every CTA once per barrier-separated
// segment of the kernel: in pass p every thread runs from the start and returns at its (p+1)-th __syncthreads(), and only the
// effects of segment p (shared and global stores, atomics, recorded loads) take place; the other segments run dry.  So each
// segment sees the complete effects of the one before it, as on the GPU.  The address of each 4-byte pixel that a global pixel load
// or store touches is recorded (a 16-byte access records its four pixels).
#include "cuda_emu.h"

#include <cstddef>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/ifb200.h"
#include "../../imageflow_b200/csrc/ifb_color.h"

namespace emu {
static int pass, seg;
static std::vector<uint64_t> loads, stores;
static bool live() { return seg == pass; }
template <class T> static void rec(std::vector<uint64_t>& v, const T* p) {
    for (size_t i = 0; i < sizeof(T) / 4; ++i) v.push_back((uint64_t)(uintptr_t)p + 4 * i);
}
template <class T> static T load(const T* p) {
    if (live()) rec(loads, p);
    return *p;
}
template <class T> static void store(T* p, const T& v) {
    if (!live()) return;
    rec(stores, p);
    *p = v;
}
template <class T, class U> static void set(T& lhs, const U& v) {
    if (live()) lhs = v;
}
template <class T> static T add(T* p, T v) {
    const T o = *p;
    if (live()) *p = o + v;
    return o;
}
}  // namespace emu
#define __shared__ static
#define __syncthreads() do { if (emu::seg == emu::pass) return; ++emu::seg; } while (0)
#define IFB_CL_LOAD4(p) emu::load(p)
#define IFB_CL_STORE4(p, v) emu::store(p, (uint32_t)(v))
#define IFB_CL_LOAD16(p) emu::load(p)
#define IFB_CL_STORE16(p, v) emu::store(p, (uint4)(v))
#define IFB_CL_SET(lhs, v) emu::set((lhs), (v))
#define IFB_CL_SHARED_ADD(p, v) emu::add((p), (v))
#define IFB_CL_GLOBAL_ADD(p, v) emu::add((p), (v))

namespace ifbk {
#include "../../imageflow_b200/csrc/ifb_types.cuh"
#include "../../imageflow_b200/csrc/ifb_color_kernel.cuh"
}  // namespace ifbk

namespace {
void run_ctas(void (*kernel)(ifbk::ClDev), const ifbk::ClDev& a, uint64_t ctas, int passes, unsigned threads) {
    for (uint64_t b = 0; b < ctas; ++b) {
        emu::blockIdx = {(unsigned)b, 0, 0};
        for (emu::pass = 0; emu::pass < passes; ++emu::pass)
            for (unsigned t = 0; t < threads; ++t) {
                emu::threadIdx = {t, 0, 0};
                emu::seg = 0;
                kernel(a);
            }
    }
}
}  // namespace

// One call of ifb200_batch_color_chain over d[0..n) as the engine makes it: color_prepare, which color_chain_locked (ifb_engine.cu)
// calls too, then the histogram, maps and apply launches (the first two only when a job white-balances).
// loads / stores receive the address of every pixel access, in order (capacity cap each; *n_loads / *n_stores = the counts);
// hist receives the 768 counters of each white balance as the histogram launch left them (capacity hist_cap counters; *n_wb = the
// white balances).  *launches = the kernel launches.  Returns the CTAs launched, or -(ifb200_status) when a descriptor is rejected
// (err = why).
// sabotage != 0 corrupts the plan before the launches, to show that the checks of the tests catch it: 1 moves the first CTA of the
// second job to the first job (a tile crossing a job), 2 points the first job at the next table (a wrong table offset), 3 points the
// first white balance at the second one's counters.
extern "C" long emu_color(const ifb200_color_desc* d, size_t n, uint64_t* loads, uint64_t* stores, size_t cap, size_t* n_loads,
                          size_t* n_stores, uint64_t* hist, size_t hist_cap, size_t* n_wb, int* launches, char* err, size_t err_cap,
                          int sabotage) {
    *launches = 0; *n_wb = 0; *n_loads = 0; *n_stores = 0;
    ifb::ClWork wk;
    int code = 0;
    const std::string why = ifb::color_prepare(d, n, wk, &code);
    if (!why.empty()) {
        snprintf(err, err_cap, "%s", why.c_str());
        return -code;
    }
    if (wk.jobs.empty()) return 0;
    if (sabotage == 1 && wk.jobs.size() > 1) --wk.first[1];
    if (sabotage == 2) ++wk.jobs[0].tab0;
    if (sabotage == 3 && wk.wb_jobs.size() > 1) wk.wb_jobs[0].wb = 1;
    std::vector<unsigned long long> counters(wk.wb_jobs.size() * 768, 0ull);
    ifbk::ClDev a{wk.jobs.data(), wk.first.data(), (uint32_t)wk.jobs.size(), wk.segs.data(), wk.tables.data(), wk.mats.data(), counters.data()};
    emu::loads.clear(); emu::stores.clear();
    uint64_t ctas = 0;
    if (!wk.wb_jobs.empty()) {
        ifbk::ClDev w = a;
        w.jobs = wk.wb_jobs.data(); w.first = wk.wb_first.data(); w.n = (uint32_t)wk.wb_jobs.size();
        run_ctas(ifbk::color_hist_kernel, w, wk.wb_ctas(), 3, ifb::kClThreads);
        for (size_t i = 0; i < counters.size() && i < hist_cap; ++i) hist[i] = counters[i];
        run_ctas(ifbk::color_maps_kernel, w, w.n, 1, 256);
        ctas += wk.wb_ctas() + w.n;
        *launches += 2;
    }
    run_ctas(ifbk::color_apply_kernel, a, wk.ctas(), 2, ifb::kClThreads);
    ctas += wk.ctas();
    *launches += 1;
    *n_wb = wk.wb_jobs.size();
    *n_loads = emu::loads.size(); *n_stores = emu::stores.size();
    for (size_t i = 0; i < emu::loads.size() && i < cap; ++i) loads[i] = emu::loads[i];
    for (size_t i = 0; i < emu::stores.size() && i < cap; ++i) stores[i] = emu::stores[i];
    return (long)ctas;
}

// The plan alone: its upload in bytes, the jobs that write pixels, the apply launch's CTAs and each job's segment kinds (kinds[i] =
// the kinds of all jobs' segments in order, capacity kinds_cap).  -1 when a descriptor is rejected.
extern "C" long emu_color_plan(const ifb200_color_desc* d, size_t n, size_t* bytes, size_t* n_jobs, uint32_t* kinds, size_t kinds_cap,
                               size_t* n_segs) {
    ifb::ClWork wk;
    int code = 0;
    if (!ifb::color_prepare(d, n, wk, &code).empty()) return -1;
    *bytes =wk.bytes(); *n_jobs = wk.jobs.size(); *n_segs = wk.segs.size();
    for (size_t i = 0; i < wk.segs.size() && i < kinds_cap; ++i) kinds[i] = wk.segs[i].kind;
    return (long)wk.ctas();
}

// The tables of a plan (for the planner tests): every table of every job in order, 1024 bytes each (capacity cap bytes).
extern "C" long emu_color_tables(const ifb200_color_desc* d, size_t n, uint8_t* out, size_t cap) {
    ifb::ClWork wk;
    int code = 0;
    if (!ifb::color_prepare(d, n, wk, &code).empty()) return -1;
    memcpy(out, wk.tables.data(), std::min(cap, wk.tables.size()));
    return (long)wk.tables.size();
}
