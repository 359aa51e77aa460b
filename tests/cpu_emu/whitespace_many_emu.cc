// Executes the batched detect_content of imageflow_b200/csrc/ifb_whitespace_kernel.cuh -- whitespace_segments_kernel and
// whitespace_walk_kernel, the product's CUDA source, unmodified -- on the CPU, with the product's host planner (ifb_whitespace.cc,
// linked as it is).  TEST INFRASTRUCTURE: nothing in the product calls it.
//   segments: sequential.  Barriers are emulated as in color_kernel_emu.cc: every CTA runs once per barrier-separated segment, and in
//     pass p only the stores of segment p take place (IFB_WS_SET), so each segment sees the complete effects of the one before it.
//   walk: the 32 lanes of a frame's warp on OS threads of their own, __syncwarp and __reduce_min_sync through a per-warp barrier
//     and exchange defined below; frames one after another.
// The summaries lie between two runs of sentinel words, and start filled with 0xA5 bytes, which no summary byte can be.
#include "cuda_emu.h"

#include <barrier>
#include <cstddef>
#include <cstdio>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include "../../include/ifb200.h"
#include "../../imageflow_b200/csrc/ifb_whitespace.h"

namespace emu {
// The walk's warp-synchronous built-ins: each lane's OS thread points `warp` at its warp's barrier and exchange slots before it
// calls the kernel.
struct Warp { std::barrier<>* bar; uint32_t slot[32]; };
static thread_local Warp* warp;
static int pass, seg;                                   // pass < 0: every store takes place (the walk)
static bool live() { return pass < 0 || seg == pass; }
template <class T, class U> static void set(T& lhs, const U& v) {
    if (live()) lhs = v;
}
}  // namespace emu
static inline void __syncwarp(unsigned = 0xffffffffu) { emu::warp->bar->arrive_and_wait(); }
static inline unsigned __reduce_min_sync(unsigned, unsigned v) {
    emu::Warp& w = *emu::warp;
    w.slot[threadIdx.x & 31] = v;
    w.bar->arrive_and_wait();
    unsigned m = ~0u;
    for (unsigned i = 0; i < 32; ++i) m = std::min(m, w.slot[i]);
    w.bar->arrive_and_wait();
    return m;
}
#define __shared__ static
#define __syncthreads() do { if (emu::seg == emu::pass) return; ++emu::seg; } while (0)
#define IFB_WS_SET(lhs, v) emu::set((lhs), (v))
#define IFB_WS_BATCH_EMU 1

namespace ifbk {
#include "../../imageflow_b200/csrc/ifb_whitespace_kernel.cuh"
}  // namespace ifbk

namespace {
constexpr size_t kGuard = 64;                           // sentinel words on each side of the summaries
constexpr uint32_t kSentinel = 0x5e5e5e5eu;
}  // namespace

// One call of ifb200_batch_detect_content_many over d[0..n) as the engine makes it: detect_content_prepare, which
// detect_content_many_locked (ifb_engine.cu) calls too, the segments launch, the walk launch.  rects (4 per job) and visited receive the
// results.  *launches = the kernel launches, *bad = frames whose walk met a window the summaries cannot replay, *guards_ok = 1 when
// every sentinel word is intact, *unwritten = summary bytes still 0xA5.  Returns the CTAs of the segments launch, or -(status) when a
// descriptor is rejected (err = why).
extern "C" long emu_detect_content_many(const ifb200_detect_content_desc* d, size_t n, uint32_t* rects, uint64_t* visited, int* launches,
                                        int* bad, int* guards_ok, uint64_t* unwritten, char* err, size_t err_cap) {
    ifb::WsWork wk;
    int code = 0;
    const std::string why = ifb::detect_content_prepare(d, n, wk, &code, rects, visited);
    if (!why.empty()) {
        snprintf(err, err_cap, "%s", why.c_str());
        return -code;
    }
    *launches = 0; *bad = 0;
    std::vector<uint32_t> mem(wk.n_sums + 2 * kGuard, kSentinel);
    uint32_t* sums = mem.data() + kGuard;
    std::memset(sums, 0xA5, wk.n_sums * 4);
    const uint64_t ctas = wk.ctas();
    if (ctas) {
        ++*launches;
        emu::gridDim = {(unsigned)ctas, 1, 1};
        for (uint64_t b = 0; b < ctas; ++b) {
            emu::blockIdx = {(unsigned)b, 0, 0};
            for (emu::pass = 0; emu::pass < 3; ++emu::pass)
                for (unsigned ty = 0; ty < ifb::kWsBand; ++ty)
                    for (unsigned tx = 0; tx < ifb::kWsChunk; ++tx) {
                        emu::threadIdx = {tx, ty, 0};
                        emu::seg = 0;
                        ifbk::whitespace_segments_kernel(wk.segs.data(), wk.first.data(), (uint32_t)wk.segs.size(), sums);
                    }
        }
    }
    std::vector<ifb::WsResult> res(wk.jobs.size());
    if (!wk.jobs.empty()) {
        ++*launches;
        emu::pass = -1;
        for (size_t k = 0; k < wk.jobs.size(); ++k) {
            emu::blockIdx = {(unsigned)k, 0, 0};
            std::barrier<> bar(32);
            emu::Warp warp{&bar, {}};
            std::vector<std::thread> th;
            for (unsigned t = 0; t < 32; ++t)
                th.emplace_back([&, t] {
                    emu::threadIdx = {t, 0, 0};
                    emu::warp = &warp;
                    ifbk::whitespace_walk_kernel(wk.jobs.data(), wk.cols.data(), sums, res.data());
                });
            for (auto& x : th) x.join();
        }
    }
    *guards_ok = 1;
    for (size_t i = 0; i < kGuard; ++i)
        if (mem[i] != kSentinel || mem[kGuard + wk.n_sums + i] != kSentinel) *guards_ok = 0;
    *unwritten = 0;
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(sums);
    for (uint64_t i = 0; i < wk.n_sums * 4; ++i) *unwritten += bytes[i] == 0xA5;
    for (size_t k = 0; k < res.size(); ++k) {
        const uint32_t i = wk.job_of[k];
        *bad += res[k].bad != 0;
        for (int q = 0; q < 4; ++q) rects[4 * i + q] = res[k].rect[q];
        if (visited) visited[i] = res[k].visited;
    }
    return (long)ctas;
}

// The plan alone: per frame that needs a walk, its grid {w, h, y1, y2, wh, rows, ncols} and its columns {bx, ex, xa, xb} into cols
// (capacity cap_cols columns).  Returns the number of such frames, or -(status) when a descriptor is rejected.
extern "C" long emu_detect_content_plan(const ifb200_detect_content_desc* d, size_t n, uint32_t* grids, uint32_t* cols, size_t cap_cols,
                                        size_t* n_cols) {
    ifb::WsWork wk;
    int code = 0;
    if (!ifb::detect_content_prepare(d, n, wk, &code, nullptr, nullptr).empty()) return -code;
    for (size_t k = 0; k < wk.jobs.size(); ++k) {
        const ifb::WsJob& j = wk.jobs[k];
        const uint32_t g[7] = {j.w, j.h, j.y1, j.y2, j.wh, j.rows, j.ncols};
        for (int q = 0; q < 7; ++q) grids[7 * k + q] = g[q];
    }
    *n_cols = wk.cols.size();
    for (size_t c = 0; c < wk.cols.size() && c < cap_cols; ++c) {
        cols[4 * c] = wk.cols[c].bx; cols[4 * c + 1] = wk.cols[c].ex; cols[4 * c + 2] = wk.cols[c].xa; cols[4 * c + 3] = wk.cols[c].xb;
    }
    return (long)wk.jobs.size();
}
