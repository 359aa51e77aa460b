// Executes imageflow_b200/csrc/ifb_orient_kernel.cuh -- the product's CUDA source, unmodified -- on the CPU under a sequential
// emulation of the few CUDA built-ins it uses, with the product's host planner (ifb_orient.cc, linked as it is).
// TEST INFRASTRUCTURE: nothing in the product calls it.  The kernel has one __syncthreads(), emulated as in whitespace_kernel_emu.cc
// by running every CTA twice: pass 0 returns at the barrier (the shared tile gets filled) and is a dry run for CTAs that have no
// barrier (global stores are dropped, no access is recorded); pass 1 runs through and records the address of each 4-byte pixel
// every global load and store touches (a 16-byte access records its four pixels).  Shared-memory indices outside the
// kOrTileOx x 32 tile are counted.
#include "cuda_emu.h"

#include <cstddef>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/ifb200.h"
#include "../../imageflow_b200/csrc/ifb_orient.h"

namespace emu {
static int pass;
static long bad_smem;
static std::vector<uint64_t> loads, stores;
template <class T> static void rec(std::vector<uint64_t>& v, const T* p) {
    for (size_t i = 0; i < sizeof(T) / 4; ++i) v.push_back((uint64_t)(uintptr_t)p + 4 * i);
}
template <class T> static T load(const T* p) {
    if (pass == 1) rec(loads, p);
    return *p;
}
template <class T> static void store(T* p, const T& v) {
    if (pass == 0) return;
    rec(stores, p);
    *p = v;
}
static uint32_t smem_dummy;
static uint32_t& smem(uint32_t (*t)[33], uint32_t r, uint32_t c) {
    if (r >= ifb::kOrTileOx || c >= 32) {
        ++bad_smem;
        return smem_dummy;
    }
    return t[r][c];
}
}  // namespace emu
#define __shared__ static
#define __syncthreads() do { if (emu::pass == 0) return; } while (0)
#define IFB_OR_LOAD4(p) emu::load(p)
#define IFB_OR_STORE4(p, v) emu::store(p, (uint32_t)(v))
#define IFB_OR_LOAD16(p) emu::load(p)
#define IFB_OR_STORE16(p, v) emu::store(p, (uint4)(v))
#define IFB_OR_TILE(t, r, c) emu::smem((t), (r), (c))

namespace ifbk {
#include "../../imageflow_b200/csrc/ifb_orient_kernel.cuh"
}  // namespace ifbk

// One call of ifb200_batch_orient over d[0..n) as the engine makes it: orient_prepare, which orient_locked (ifb_engine.cu) calls too,
// then one launch.  loads / stores receive the address of every pixel access, in order (capacity cap each;
// *n_loads / *n_stores = the counts), *bad_smem the shared-memory indices outside the tile.  Returns the number of CTAs launched,
// or -1 when a descriptor is rejected (err = why).  *n_items = the work items planned.
// sabotage != 0 corrupts the plan before the launch, to show that the checks of the tests catch it: 1 toggles the x reversal of
// the first item (a neighbouring orientation), 2 moves the first item's output one pixel to the right, 3 drops the last CTA.
extern "C" long emu_orient(const ifb200_orient_desc* d, size_t n, uint64_t* loads, uint64_t* stores, size_t cap, size_t* n_loads,
                           size_t* n_stores, long* bad_smem, size_t* n_items, char* err, size_t err_cap, int sabotage) {
    ifb::OrWork wk;
    int code = 0;
    const std::string why = ifb::orient_prepare(d, n, wk, &code);
    if (!why.empty()) {
        snprintf(err, err_cap, "%s", why.c_str());
        return -1;
    }
    *n_items = wk.items.size();
    uint64_t ctas = wk.ctas();
    if (sabotage == 1 && !wk.items.empty()) wk.items.front().flags ^= ifb::kOrFx;
    if (sabotage == 2 && !wk.items.empty()) wk.items.front().out += 4;
    if (sabotage == 3 && ctas) --ctas;
    emu::loads.clear(); emu::stores.clear(); emu::bad_smem = 0;
    for (unsigned b = 0; b < ctas; ++b) {
        emu::blockIdx = {b, 0, 0};
        for (emu::pass = 0; emu::pass < 2; ++emu::pass)
            for (unsigned t = 0; t < ifb::kOrThreads; ++t) {
                emu::threadIdx = {t, 0, 0};
                ifbk::orient_kernel(wk.items.data(), wk.first.data(), (uint32_t)wk.items.size());
            }
    }
    *n_loads = emu::loads.size(); *n_stores = emu::stores.size(); *bad_smem = emu::bad_smem;
    for (size_t i = 0; i < emu::loads.size() && i < cap; ++i) loads[i] = emu::loads[i];
    for (size_t i = 0; i < emu::stores.size() && i < cap; ++i) stores[i] = emu::stores[i];
    return (long)ctas;
}

// The plan alone: the number of work items and CTAs of one call (-1 when a descriptor is rejected).
extern "C" long emu_orient_plan(const ifb200_orient_desc* d, size_t n, size_t* n_items) {
    ifb::OrWork wk;
    int code = 0;
    if (!ifb::orient_prepare(d, n, wk, &code).empty()) return -1;
    *n_items = wk.items.size();
    return (long)wk.ctas();
}
