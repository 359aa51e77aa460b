// ifb_canvas_kernel.cuh -- included by ifb_kernels.cuh inside namespace ifbk (product code, sm_90a).  Uses only threadIdx, blockIdx
// and uint4 -- tests/cpu_emu/canvas_kernel_emu.cc compiles this file with g++ under a sequential emulation of those and checks it
// against the oracle.
//
// The canvas operations of ifb200_batch_canvas, planned on the host into disjoint rectangle work items (ifb_canvas.h): one thread per
// 16-byte group of a row of an item.  Groups are aligned to the destination's addresses; a full group whose source (for a copy) is
// 16-byte aligned too moves as one 16-byte access, every other pixel as a 4-byte word.  Nothing outside an item's rectangle is read
// or written, so stride padding and neighbouring windows stay untouched.  Loads come only from copy sources and from pixels
// normalised in place.  No shared memory: the op is bound by HBM.
#ifndef IFB_CV_LOAD4                                             // the CPU emulation defines these to record every pixel access
#define IFB_CV_LOAD4(p) (*(p))
#define IFB_CV_STORE4(p, v) (*(p) = (v))
#define IFB_CV_LOAD16(p) (*(p))
#define IFB_CV_STORE16(p, v) (*(p) = (v))
#endif

__device__ __forceinline__ void cv_group(const ifb::CvItem& it, uint32_t row, uint32_t g) {
    uint8_t* const drow = it.dst + (size_t)row * it.dst_stride;
    const uint32_t a = (uint32_t)((reinterpret_cast<uintptr_t>(drow) & 15) >> 2);      // the row's first pixel is word a of its group
    const uint32_t lo = max(4 * g, a) - a, hi = min(4 * g + 4, a + it.w) - a;         // pixels [lo, hi) of the row
    if (lo >= hi) return;
    uint32_t* const d = reinterpret_cast<uint32_t*>(drow) + lo;
    const uint32_t or_a = (it.kind == ifb::kCvOpaque || (it.flags & ifb::kCvOrAlpha)) ? 0xFF000000u : 0u;
    uint32_t* const s = it.kind == ifb::kCvCopy ? reinterpret_cast<uint32_t*>(it.src + (size_t)row * it.src_stride) + lo : d;
    const bool wide = hi - lo == 4 && (reinterpret_cast<uintptr_t>(s) & 15) == 0;
    if (it.kind == ifb::kCvFill) {
        if (wide) IFB_CV_STORE16(reinterpret_cast<uint4*>(d), make_uint4(it.color, it.color, it.color, it.color));
        else for (uint32_t i = 0; i < hi - lo; ++i) IFB_CV_STORE4(d + i, it.color);
        return;
    }
    const bool back = (it.flags & ifb::kCvWriteBack) != 0;
    if (wide) {
        uint4 v = IFB_CV_LOAD16(reinterpret_cast<const uint4*>(s));
        v.x |= or_a; v.y |= or_a; v.z |= or_a; v.w |= or_a;
        IFB_CV_STORE16(reinterpret_cast<uint4*>(d), v);
        if (back) IFB_CV_STORE16(reinterpret_cast<uint4*>(s), v);
    } else {
        for (uint32_t i = 0; i < hi - lo; ++i) {
            const uint32_t v = IFB_CV_LOAD4(s + i) | or_a;
            IFB_CV_STORE4(d + i, v);
            if (back) IFB_CV_STORE4(s + i, v);
        }
    }
}

__global__ void __launch_bounds__(256) canvas_kernel(const ifb::CvItem* __restrict__ items, const ifb::CvTile* __restrict__ tiles) {
    const ifb::CvTile t = tiles[blockIdx.x];
    const ifb::CvItem it = items[t.item];
    for (uint32_t i = threadIdx.x; i < t.count; i += ifb::kCvThreads) {
        const uint32_t k = t.first + i;
        cv_group(it, k / it.groups, k % it.groups);
    }
}
