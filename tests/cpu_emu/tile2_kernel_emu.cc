// Runs imageflow_b200/csrc/ifb_tile2_kernel.cuh -- the product's CUDA source of fused_tile2_kernel, unmodified -- on the CPU:
// one OS thread per CUDA thread of a block, std::barrier for __syncthreads, a per-warp exchange for __reduce_max_sync, the CUDA
// arithmetic intrinsics mapped onto IEEE host operations (cuda_emu.h; built with -ffp-contract=off; the rounding mode stays
// round-to-nearest, and __fadd_rz / __float2uint_rz round toward zero in software).  Blocks of the grid
// run one after the other.  Dynamic shared memory is an exactly-sized heap block and every global buffer is whatever the
// caller allocated, so building this file with -fsanitize=address turns a run into a memory check of the kernel.
// TEST INFRASTRUCTURE: nothing in the product calls this; the GPU remains the place where the kernel is run and timed.
#include "cuda_emu.h"

#include <barrier>
#include <cstddef>
#include <cstdlib>
#include <memory>
#include <thread>
#include <vector>

namespace emu {
static unsigned char* smem;
static std::barrier<>* block_barrier;
static std::barrier<>* warp_barrier[8];
static unsigned warp_scratch[8][32];
}  // namespace emu
#define IFB_DYNAMIC_SMEM(name_) unsigned char* const name_ = emu::smem
#define __syncthreads() emu::block_barrier->arrive_and_wait()
static inline unsigned __reduce_max_sync(unsigned, unsigned v) {
    const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    emu::warp_scratch[warp][lane] = v;
    emu::warp_barrier[warp]->arrive_and_wait();
    unsigned m = 0;
    for (int i = 0; i < 32; ++i) m = std::max(m, emu::warp_scratch[warp][i]);
    emu::warp_barrier[warp]->arrive_and_wait();
    return m;
}

namespace ifbk {
#include "../../imageflow_b200/csrc/ifb_types.cuh"
#ifndef IFB_TILE2_MINB
#define IFB_TILE2_MINB 4
#endif
#include "../../imageflow_b200/csrc/ifb_tile2_kernel.cuh"
}  // namespace ifbk

using namespace ifbk;
using KernelFn = void (*)(const JobDev*, uint32_t, Tables, AxisDev, AxisDev, TilePlanDev);
static KernelFn pick(int ch, int linear, int compose, int cm) {
#define IFB_PICK(CH_, LIN_, CO_, CM_) if (ch == CH_ && linear == LIN_ && compose == CO_ && cm == CM_) return fused_tile2_kernel<CH_, LIN_ != 0, CO_, CM_ != 0>;
#define IFB_PICK_CM(CH_, LIN_, CO_) IFB_PICK(CH_, LIN_, CO_, 0) IFB_PICK(CH_, LIN_, CO_, 1)
#define IFB_PICK_LIN(CH_, CO_) IFB_PICK_CM(CH_, 0, CO_) IFB_PICK_CM(CH_, 1, CO_)
    IFB_PICK_LIN(4, 0) IFB_PICK_LIN(4, 1) IFB_PICK_LIN(4, 2) IFB_PICK_LIN(3, 0)
    return nullptr;
}

extern "C" uint32_t emu_tile2_smem_bytes(int max_ir, int max_ic, int linear) { return Tile2Smem::make(max_ir, max_ic, linear != 0).total; }
extern "C" int emu_tile2_tile_h(void) { return kTile2H; }
extern "C" uint32_t emu_tile2_sizeof_jobdev(void) { return (uint32_t)sizeof(JobDev); }

// one launch of fused_tile2_kernel<ch, linear, compose, cm> with `grid` blocks of 256 threads
extern "C" int emu_tile2_launch(int ch, int linear, int compose, int cm, unsigned grid, const void* jobs, uint32_t n_jobs,
                                const float* t_lin, const float* t_srgb, const uint8_t* lut16k,
                                const uint32_t* v_left, const uint32_t* v_right, const uint32_t* v_off, const float* v_w,
                                const uint32_t* h_left, const uint32_t* h_right, const uint32_t* h_off, const float* h_w,
                                const int32_t* plan10, const float* tile_vw, const uint32_t* tile_vq, const float* tile_hw) {
    KernelFn fn = pick(ch, linear, ch == 4 ? compose : 0, cm);
    if (!fn) return 1;
    TilePlanDev pl{};
    pl.in_w = (uint32_t)plan10[0]; pl.in_h = (uint32_t)plan10[1]; pl.out_w = (uint32_t)plan10[2]; pl.out_h = (uint32_t)plan10[3];
    pl.tow = plan10[4]; pl.toh = plan10[5]; pl.tiles_x = plan10[6]; pl.tiles_y = plan10[7]; pl.max_ic = plan10[8]; pl.max_ir = plan10[9];
    pl.h4 = plan10[10]; pl.vw = tile_vw; pl.vq = tile_vq; pl.hw = tile_hw;
    const Tables tb{t_lin, t_srgb, lut16k};
    const AxisDev av{v_left, v_right, v_off, v_w}, ah{h_left, h_right, h_off, h_w};
    const size_t smem_bytes = Tile2Smem::make(pl.max_ir, pl.max_ic, linear != 0).total;
    emu::gridDim = {grid, 1, 1};
    for (unsigned b = 0; b < grid; ++b) {
        emu::blockIdx = {b, 0, 0};
        // exactly sized (Tile2Smem::total is a multiple of 16) and filled with NaN patterns: an access past the end is an
        // AddressSanitizer report, and uninitialised shared memory can never pass for a result
        std::unique_ptr<unsigned char, decltype(&std::free)> sm(static_cast<unsigned char*>(std::aligned_alloc(16, smem_bytes)), &std::free);
        std::memset(sm.get(), 0xFF, smem_bytes);
        emu::smem = sm.get();
        std::barrier<> bb(256);
        emu::block_barrier = &bb;
        std::vector<std::unique_ptr<std::barrier<>>> wb;
        for (int w = 0; w < 8; ++w) { wb.emplace_back(new std::barrier<>(32)); emu::warp_barrier[w] = wb.back().get(); }
        std::vector<std::thread> th;
        for (unsigned t = 0; t < 256; ++t)
            th.emplace_back([=] {
                emu::threadIdx = {t, 0, 0};
                fn(static_cast<const JobDev*>(jobs), n_jobs, tb, av, ah, pl);
            });
        for (auto& x : th) x.join();
        emu::block_barrier = nullptr;
    }
    return 0;
}
