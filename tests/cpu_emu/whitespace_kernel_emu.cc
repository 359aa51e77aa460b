// Executes imageflow_b200/csrc/ifb_whitespace_kernel.cuh -- the product's CUDA source, unmodified -- on the CPU under a
// sequential emulation of the few CUDA built-ins it uses.  TEST INFRASTRUCTURE: it checks indexing and arithmetic of a
// kernel before (and in addition to) its runs on a GPU; nothing in the product calls it.
//   threads of a block run one after the other; the kernel has ONE __syncthreads(), which is emulated by running every
//   thread twice: pass 0 returns at the barrier (the shared tile gets filled), pass 1 runs through (each thread rewrites
//   the same tile values, then computes its pixel).
#include "cuda_emu.h"

namespace emu {
static int pass;
}  // namespace emu
#define __shared__ static
#define __syncthreads() do { if (emu::pass == 0) return; } while (0)

namespace ifbk {
#include "../../imageflow_b200/csrc/ifb_whitespace_kernel.cuh"
}

extern "C" void emu_whitespace_codes(const uint8_t* px, uint32_t w, uint32_t h, uint32_t stride, uint32_t alpha_meaningful, int threshold, uint8_t* codes) {
    const unsigned gx = (w + 31) / 32, gy = (h + 7) / 8;                 // the launch configuration of detect_content_locked (ifb_engine.cu)
    for (unsigned by = 0; by < gy; ++by)
        for (unsigned bx = 0; bx < gx; ++bx) {
            emu::blockIdx = {bx, by, 0};
            for (emu::pass = 0; emu::pass < 2; ++emu::pass)
                for (unsigned ty = 0; ty < 8; ++ty)
                    for (unsigned tx = 0; tx < 32; ++tx) {
                        emu::threadIdx = {tx, ty, 0};
                        ifbk::whitespace_codes_kernel(px, w, h, stride, alpha_meaningful, threshold, codes, 0u);
                    }
        }
}
