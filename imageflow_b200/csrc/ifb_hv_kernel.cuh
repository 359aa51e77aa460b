// ifb_hv_kernel.cuh -- the hot kernel of the resample path (product code, sm_90a); included by ifb_kernels.cuh inside namespace ifbk.
//
// Stands in for zenresize's StreamingResize behind graphics/scaling.rs:93-251: rows stream in, every row is filtered
// horizontally as it arrives, output rows are emitted as soon as their vertical window is complete.  Down-scales (and 1:1)
// whose contribution windows keep at most AV <= 6 outputs open per source sample on both axes run here.
//
// Decomposition: ONE WARP = one work item = (job, strip of output columns, band of output rows), and inside it LANE = SOURCE ROW.
// A warp walks its band 32 source rows at a time ("row block"); for every row block it streams the strip's source columns left to right:
//   * TMA (cp.async.bulk.tensor.2d, SWIZZLE_64B) stages one box of 16 pixels x 32 rows into the warp's own shared-memory ring
//     (kStages deep, one mbarrier per stage; the same warp issues, waits and consumes: no other synchronisation exists in this
//     kernel).  The 64-byte swizzle makes the per-lane 16-byte reads of "my row" bank-conflict free.
//   * H pass: every lane converts its pixel through the lane-replicated LUT (one PRMT + one conflict-free LDS per channel) and
//     multiply-adds it into a ring of AV accumulators: output column X owns slot X mod AV while its window is open.  The weights
//     of a source column are the same for all lanes: one broadcast LDS.128 per source column of a table the CTA keeps in shared
//     memory.  The whole horizontal reduction (7.5 : 1 for 4K -> 512) happens in registers with no exchange between threads; what
//     steers it (which column completes where) is warp-uniform.
//   * When a column completes, its CH values go to the warp's exchange buffer [column][channel][row]; after kCG columns (a "group")
//     the warp turns around: LANE = (pair of ring slots, OUTPUT COLUMN), and the 32 H-filtered rows of the block are multiply-added,
//     in row order, into the group's vertical accumulators (output row Y owns slot Y mod AV; a lane holds two of the AV slots of
//     its column as one packed pair, so the 32 lanes do AV/2 x kCG columns).  A completed output row goes through the store
//     epilogue in the lanes that hold its slot and is written as one coalesced segment.
// One 32-row stream per warp and as many warps as shared memory holds (16, or 12 with four channels): the first form of this
// kernel gave every lane two streams in half as many warps; at two warps per scheduler every branch, instruction-cache miss and
// fixed latency was exposed.
// Every source pixel is read from HBM once (plus strip/band halos), converted once; nothing but source and destination
// pixels touches HBM.  Arithmetic: the H chain ascends over source columns from +0, the V chain over source rows from +0 --
// exactly the order of the specification (DESIGN.md section 3); a slot only ever sees zero weights outside its window, and fmaf(+0, v, acc) == acc.
//
// Shared memory (one CTA per SM, kWarps warps):
//   LUT block, 64 KB, placed so that its shared-window address is a multiple of 64 KB (the layout adapts to wherever the
//   driver puts dynamic shared memory): row v (256 B): bytes 0..127 = T[v] for the 32 lanes, so the window address of a lookup
//   is LUT | v << 8 | lane << 2 -- one PRMT, bank-conflict free for any image content.  Bytes 128..255 of the rows ("holes"):
//   holes 0..127 = the 16 KB linear->sRGB table of the store epilogue, holes 128..255 = the strip's H weights (16 KB).
//   Around it, per warp: stage ring, exchange buffer, mbarriers (hv_layout() packs them into the space before and after the LUT block).
#pragma once

#include "ifb_profile_step.cuh"

#ifndef IFB_HV_EMU
#include <cuda.h>          // CUtensorMap (type only; the driver entry point is looked up at run time by the engine)
#endif

struct HvStripDev { int X0, X1, Xf, hslot0, k0, nst, pad0, pad1; };   // columns [X0,X1); first completing column Xf (<= X0) and its slot;
                                                                      // pixel stream = source columns k0 .. k0 + 16*nst - 1
struct HvBandDev  { int Y0, Y1, Yf, vslot0, j0, nrows, pad0, pad1; }; // rows [Y0,Y1); first completing row Yf and its slot; source rows j0 .. j0+nrows-1
struct HvPlanDev {
    uint32_t in_w, in_h, out_w, out_h;
    int n_strips, n_bands;
    const HvStripDev* strips;
    const HvBandDev* bands;
    const float* hw;          // [n_strips][hw_stride][AVP]: weight of the open output column in each ring slot, pixel-stream order (the
                              // kernel stages each record in register order: ifb_hv_ring_body.inc, H weights of the strip)
    const uint8_t* hdone;     // [n_strips][hw_stride + 64]: output columns completing after this pixel (bits 0..6), V-pass mark (bit 7)
    const float* vw;          // [in_h][AVP]
    const uint8_t* vdone;     // [in_h + 32]
    uint32_t zero;            // 0 (a zero the compiler cannot see: hv::zero_after)
    uint32_t hw_stride;       // source columns (weight records) per strip in hw; hdone has hw_stride + 64 bytes per strip
};
struct alignas(64) HvTmap { unsigned char bytes[128]; };              // CUtensorMap of one job's input bitmap (u32 pixels, box 16 x 32, SWIZZLE_64B;
                                                                      // oriented flags 5..8: box 32 x 16, no swizzle)
// What a ring kernel instantiation reads (template parameter ORI): the stored frame (0); flags 2..4, the box of the stored frame with
// either axis walked backwards (1); flags 5..8, the transposed box, the lanes along source columns (2).  Which axes run backwards is
// per job (JF_FLIP_X / JF_FLIP_Y).
enum : int { HV_ORI_NONE = 0, HV_ORI_FLIP = 1, HV_ORI_TRANSPOSE = 2 };
// The source pixel format an instantiation reads (template parameter SRC, ifb200_batch_enqueue_rows): BGRA32 (0); RGBA32 (1), the
// same u32 box, the table look-ups taking blue from byte 2 and red from byte 0; RGB24 (2), a UINT8 tensor read in boxes of 64 bytes
// x 32 rows, 16 pixels (48 bytes) at a constant offset r inside each box (transposed: boxes of 128 bytes x 16 rows, 32 pixels at r).
enum : int { HV_SRC_BGRA = 0, HV_SRC_RGBA = 1, HV_SRC_RGB24 = 2 };

#ifndef IFB_HV_MAXCOLS4
#define IFB_HV_MAXCOLS4 64             // widest strip of the ring-depth-4 variants (V accumulators: 12 or 16 registers per 16 columns)
#endif
#ifndef IFB_HV_STAGES
#define IFB_HV_STAGES 2                // ring slots per warp (A/B builds: with more, fewer warps fit; DESIGN.md section 5.1)
#endif
#ifndef IFB_HV_WARPS3
#define IFB_HV_WARPS3 16               // warps per CTA with three channels
#endif
#ifndef IFB_HV_WARPS4
#define IFB_HV_WARPS4 12               // and with four
#endif
// Probe builds (A/B measurements only, never the product; their outputs are wrong on purpose):
//   IFB_HV_PROBE_MEM   the TMA stream alone: same boxes, waits and refill points; the H and V arithmetic replaced by one dependent
//                      use of each chunk's bytes, one word stored per work item
//   IFB_HV_PROBE_MATH  the arithmetic alone: H pass, V pass and store over boxes fetched once per work item (one per ring slot),
//                      then read again and again with no refill and no wait
//   IFB_HV_PROBE_NOPARK  (with IFB_HV_PROBE_MATH) every chunk with one completion runs as the plain form: the arithmetic side
//                      without the cost of parking a column (the column is counted and its place in the exchange buffer
//                      advanced; its values are never stored or cleared and the registers do not rotate)
#ifndef IFB_HV_PROBE_MEM
#define IFB_HV_PROBE_MEM 0
#endif
#ifndef IFB_HV_PROBE_MATH
#define IFB_HV_PROBE_MATH 0
#endif
#ifndef IFB_HV_PROBE_NOPARK
#define IFB_HV_PROBE_NOPARK 0
#endif
// PROF (PF_MATRIX, PF_GRAY): the forms of ifb200_batch_enqueue_profiled, which apply a profile's plan to every source pixel; its
// tables (ProfDev) take kProfBytes of shared memory, so the three-channel forms run one warp fewer at ring depth 4, and 12 warps at
// ring depth 6, where 13..16 warps leave 128 registers and seven forms spilled (DESIGN.md section 5.20).
template <int AV, int CH, int PROF = PF_IDENTITY> struct HvCfg {
    static_assert(AV == 4 || AV == 6, "ring depth");
    static constexpr int kAvp = AV == 4 ? 4 : 8;                      // floats per weight record
    static constexpr int kCapPx = 16384 / (kAvp * 4);                 // pixels of H weights that fit in the holes
    static constexpr int kNP = AV / 2;                                // packed slot pairs
    static constexpr int kCG = 32 / kNP;                              // output columns per group: kNP x kCG lanes in the V pass (16, or 10 at ring depth 6)
    static constexpr int kMaxCols = AV == 4 ? IFB_HV_MAXCOLS4 : (CH == 3 ? 50 : 40);   // widest strip (output columns)
    static constexpr int kNG = kMaxCols / kCG + 1;                    // column groups per strip (V accumulators: 2 * CH registers per group); groups end on
                                                                      // chunk-pair boundaries and are not always full, hence one more than the columns need
    static constexpr int kWarps = PROF == PF_IDENTITY ? (CH == 3 ? IFB_HV_WARPS3 : IFB_HV_WARPS4) : CH == 4 ? IFB_HV_WARPS4 : AV == 4 ? IFB_HV_WARPS3 - 1 : 12;
    static constexpr uint32_t kProfBytes = PROF == PF_MATRIX ? 3u * 1024u : PROF == PF_GRAY ? 256u : 0u;   // tone tables / byte map
    static constexpr int kThreads = kWarps * 32;
    static constexpr int kStages = IFB_HV_STAGES;                     // boxes in the ring: up to kStages - 1 in flight while one is read
    static constexpr int kBoxBytes = 32 * 64;                         // one box: 32 rows x 16 pixels
    static constexpr int kStageBytes = kBoxBytes;
    static constexpr int kRingBytes = kStages * kStageBytes;
    static constexpr int kXPitch = CH * 32 + 2;                       // words per column of the exchange buffer: rows are written one word per lane (any
                                                                      // pitch is conflict-free), the V pass reads two rows per access: 8-byte aligned columns
                                                                      // whose 16 (or 10) 8-byte accesses fall into different bank pairs (pitch = 2 mod 32)
    static constexpr int kXBytes = kCG * kXPitch * 4;
};

// Shared-memory packing for a given low half of the shared-window base (the LUT block must start on a 64 KB boundary of the
// window, which splits dynamic shared memory into a region before it and one after it).  Per warp: a stage ring (512-byte aligned:
// the swizzle pattern repeats every 512 bytes), an exchange buffer (16-byte aligned), kStages mbarriers.  The region before the
// LUT block takes as many rings and then exchange buffers as fill it best; the rest follows the block.  Returns the bytes of dynamic
// shared memory needed; fills the window OFFSETS (from the dynamic shared-memory base) of warp `warp`'s blocks when the pointers are given.
template <int AV, int CH, int PROF = PF_IDENTITY>
__host__ __device__ constexpr uint32_t hv_layout(uint32_t sb_low16, int warp, uint32_t* st_off, uint32_t* x_off, uint32_t* mb_off) {
    using C = HvCfg<AV, CH, PROF>;
    const uint32_t lut_off = (0x10000u - sb_low16) & 0xffffu;
    const uint32_t ring = (uint32_t)C::kRingBytes, xb = (uint32_t)C::kXBytes, W = (uint32_t)C::kWarps;
    const uint32_t a0 = (512u - (sb_low16 & 511u)) & 511u;             // first 512-byte aligned offset of the region before the block
    const uint32_t roomA = lut_off > a0 ? lut_off - a0 : 0u;
    uint32_t ra = 0, xa = 0, best = 0;                                 // rings / exchange buffers placed before the block
    for (uint32_t r = 0; r <= W; ++r) {
        if (r * ring > roomA) break;
        uint32_t x = (roomA - r * ring) / xb;
        if (x > W) x = W;
        const uint32_t used = r * ring + x * xb;
        if (used > best) { best = used; ra = r; xa = x; }
    }
    const uint32_t b0 = lut_off + 65536u;                              // window address there is a multiple of 64 KB
    const uint32_t b_x = b0 + (W - ra) * ring;                         // exchange buffers behind the block's rings
    const uint32_t b_mb = (b_x + (W - xa) * xb + 7u) & ~7u;
    if (warp >= 0) {
        const uint32_t w = (uint32_t)warp;
        if (st_off) *st_off = w < ra ? a0 + w * ring : b0 + (w - ra) * ring;
        if (x_off) *x_off = w < xa ? a0 + ra * ring + w * xb : b_x + (w - xa) * xb;
        if (mb_off) *mb_off = b_mb + w * 8u * (uint32_t)C::kStages;
    }
    return b_mb + W * 8u * (uint32_t)C::kStages + C::kProfBytes + 16u;   // + the profile's tables (hv_prof_offset) + one CTA-wide flag word (hv_flag_offset)
}
// window offset of the CTA-wide flag word: the last 16 bytes of the layout; of the profile's tables: the kProfBytes before it
template <int AV, int CH, int PROF = PF_IDENTITY> __host__ __device__ constexpr uint32_t hv_flag_offset(uint32_t sb_low16) { return hv_layout<AV, CH, PROF>(sb_low16, -1, nullptr, nullptr, nullptr) - 16u; }
template <int AV, int CH, int PROF = PF_IDENTITY> __host__ __device__ constexpr uint32_t hv_prof_offset(uint32_t sb_low16) { return hv_flag_offset<AV, CH, PROF>(sb_low16) - HvCfg<AV, CH, PROF>::kProfBytes; }
template <int AV, int CH, int PROF = PF_IDENTITY> constexpr uint32_t hv_total_bytes(uint32_t sb_low16) { return hv_layout<AV, CH, PROF>(sb_low16, -1, nullptr, nullptr, nullptr); }

// ---------------------------------------------------------------- primitives (tests/cpu_emu provides its own under IFB_HV_EMU)
#ifndef IFB_HV_EMU
namespace hv {
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// table look-ups: volatile, so that a chunk's 24 look-ups stay in its chunk (hoisted to the top of the stage they would need 96 registers)
__device__ __forceinline__ float lds_lut(uint32_t a) { float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a)); return v; }
// the look-up of byte SEL of a packed pixel: window address = PRMT(pixel, lane4, selector) = LUT | byte << 8 | lane << 2, built and used in
// one statement (the address never occupies a register beyond the load)
template <uint32_t SEL> __device__ __forceinline__ float lut_gather(uint32_t px, uint32_t lane4) {
    float v;
    asm volatile("{\n\t.reg .b32 a;\n\tprmt.b32 a, %1, %2, %3;\n\tld.shared.f32 %0, [a];\n\t}" : "=f"(v) : "r"(px), "r"(lane4), "n"(SEL));
    return v;
}
__device__ __forceinline__ uint32_t lds_lut_u8(uint32_t a) { uint32_t v; asm("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
// weight records: volatile, so that they are fetched where the chunk that uses them starts (hoisted to the top of a stage, the 16
// records of its four chunks would occupy 64 registers)
__device__ __forceinline__ float4 lds_w4(uint32_t a) {
    float4 v; asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a)); return v;
}
__device__ __forceinline__ float2 lds_w2(uint32_t a) { float2 v; asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a)); return v; }
__device__ __forceinline__ float lds_f32(uint32_t a) { float v; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory"); return v; }
__device__ __forceinline__ uint4 lds_u32x4(uint32_t a) {
    uint4 v; asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory"); return v;
}
__device__ __forceinline__ void sts_f32(uint32_t a, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory"); }
__device__ __forceinline__ void sts_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts_f32x4(uint32_t a, float4 v) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(a), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// A completed output column, without a branch: if (mask & BIT) { park a0.. at [xw], [xw + 128], ..; clear them; xw += STEP; } as
// predicated instructions behind one predicate (a branch, taken or not, holds the warp until it is resolved).
template <uint32_t BIT, uint32_t STEP>
__device__ __forceinline__ void flush3_if(uint32_t& xw, float& a0, float& a1, float& a2, const uint32_t mask) {
    asm volatile("{\n\t.reg .pred q;\n\t.reg .b32 t;\n\t"
                 "and.b32 t, %4, %5;\n\tsetp.ne.u32 q, t, 0;\n\t"
                 "@q st.shared.f32 [%0], %1;\n\t@q st.shared.f32 [%0+128], %2;\n\t@q st.shared.f32 [%0+256], %3;\n\t"
                 "@q mov.f32 %1, 0f00000000;\n\t@q mov.f32 %2, 0f00000000;\n\t@q mov.f32 %3, 0f00000000;\n\t"
                 "@q add.u32 %0, %0, %6;\n\t}"
                 : "+r"(xw), "+f"(a0), "+f"(a1), "+f"(a2) : "r"(mask), "n"(BIT), "n"(STEP) : "memory");
}
template <uint32_t BIT, uint32_t STEP>
__device__ __forceinline__ void flush4_if(uint32_t& xw, float& a0, float& a1, float& a2, float& a3, const uint32_t mask) {
    asm volatile("{\n\t.reg .pred q;\n\t.reg .b32 t;\n\t"
                 "and.b32 t, %5, %6;\n\tsetp.ne.u32 q, t, 0;\n\t"
                 "@q st.shared.f32 [%0], %1;\n\t@q st.shared.f32 [%0+128], %2;\n\t@q st.shared.f32 [%0+256], %3;\n\t@q st.shared.f32 [%0+384], %4;\n\t"
                 "@q mov.f32 %1, 0f00000000;\n\t@q mov.f32 %2, 0f00000000;\n\t@q mov.f32 %3, 0f00000000;\n\t@q mov.f32 %4, 0f00000000;\n\t"
                 "@q add.u32 %0, %0, %7;\n\t}"
                 : "+r"(xw), "+f"(a0), "+f"(a1), "+f"(a2), "+f"(a3) : "r"(mask), "n"(BIT), "n"(STEP) : "memory");
}
// 0, but only once v has arrived: v & zero with a zero that comes from the kernel's arguments, so that the instruction (and the
// scoreboard wait on v) survives.  (v ^ v is folded away by ptxas; and it also drops __syncwarp() where it knows the warp to be
// converged, so nothing else would keep a TMA refill of a ring slot behind the slot's last LDS.  Found with compute-sanitizer:
// its instrumented loads are slow enough to lose that race.)
__device__ __forceinline__ uint32_t zero_after(uint32_t v, uint32_t zero) { uint32_t z; asm volatile("and.b32 %0, %1, %2;" : "=r"(z) : "r"(v), "r"(zero)); return z; }
__device__ __forceinline__ float saturate(float v) { return __saturatef(v); }
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) { return __byte_perm(a, b, sel); }
// a packed pair of accumulators: two FFMA (sm_90 has no packed f32x2 multiply-add); each half is fmaf(a, b, c)
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ uint32_t ballot(bool p) { return __ballot_sync(0xffffffffu, p); }
__device__ __forceinline__ uint32_t bcast0(uint32_t v) { return __shfl_sync(0xffffffffu, v, 0); }
__device__ __forceinline__ uint32_t warp_sum(uint32_t v) { return __reduce_add_sync(0xffffffffu, v); }
__device__ __forceinline__ void warp_sync() { __syncwarp(); }
__device__ __forceinline__ bool elect_one() {              // true in exactly one lane of the (converged) warp
    uint32_t is_leader;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(is_leader));
    return is_leader != 0;
}
__device__ __forceinline__ void cta_sync() { __syncthreads(); }
__device__ __forceinline__ uint32_t atomic_inc(uint32_t* p) { return atomicAdd(p, 1u); }
__device__ __forceinline__ void mbar_init(uint32_t addr, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(addr), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_init_fence() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t addr, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(addr), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t addr, uint32_t parity) {
    // The retry loop lives inside the asm statement, with uniform branches: written as a C loop it made ptxas give up on the
    // warp being converged for the rest of the kernel (every vote behind a BRA.DIV, every warp-uniform branch wrapped in
    // BSSY/BSYNC).  try_wait suspends the thread for a hardware-defined time before it reports failure, so the loop is rarely
    // taken; a transfer that never completes (a bad descriptor) is given up after a few seconds instead of hanging the device (a
    // `trap` in this loop brings the convergence barriers back).
    asm volatile("{\n\t.reg .pred p;\n\t.reg .u32 n;\n\t"
                 "mov.u32 n, 0;\n\t"
                 "IFB_WAIT:\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
                 "@p bra.uni IFB_DONE;\n\t"
                 "add.u32 n, n, 1;\n\t"
                 "setp.lt.u32 p, n, 0x1000000;\n\t"
                 "@p bra.uni IFB_WAIT;\n\t"
                 "IFB_DONE:\n\t}" :: "r"(addr), "r"(parity) : "memory");
}
// one box of 16 pixels x 32 rows at pixel (x, y) of the job's bitmap -> shared memory, completion counted on the mbarrier
__device__ __forceinline__ void tma_load_box(uint32_t dst, const HvTmap* tm, int x, int y, uint32_t mbar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(tm), "r"(mbar), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void tma_prefetch_box(const HvTmap* tm, int x, int y) {
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global [%0, {%1, %2}];" ::"l"(tm), "r"(x), "r"(y) : "memory");
}
template <class T> __device__ __forceinline__ T ldg(const T* p) { return __ldg(p); }
__device__ __forceinline__ uint32_t ldg_volatile(const uint32_t* p) { return *reinterpret_cast<const volatile uint32_t*>(p); }
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory"); return v; }
}  // namespace hv
#define IFB_HV_DYNAMIC_SMEM(name_) extern __shared__ __align__(1024) unsigned char name_[]
#endif

// Where a CTA's dynamic shared memory starts in the shared window (the engine sizes the ring kernel's layout with it).
__global__ void smem_base_probe_kernel(uint32_t* out) {
    IFB_HV_DYNAMIC_SMEM(probe_smem);
    if (threadIdx.x == 0) *out = hv::smem_u32(probe_smem);
}

// The LUT block's tables, filled by threads t, t + NT, ..: forward LUT replicated for the 32 lanes; linear->sRGB table into
// holes 0..127.  Its own function so that tests/gpu_units gives hv_finish_pixel() the very layout the kernel reads.
template <int NT>
__device__ __forceinline__ void hv_fill_luts(const uint32_t lut, const Tables& tb, const uint32_t flags0, const int t) {
    const float* __restrict__ T = (flags0 & JF_LINEAR) ? tb.t_lin : tb.t_srgb;
    for (int i = t; i < 256 * 32; i += NT) hv::sts_f32(lut + ((uint32_t)(i >> 5) << 8) + ((uint32_t)(i & 31) << 2), hv::ldg(T + (i >> 5)));
    const uint32_t* __restrict__ r32 = reinterpret_cast<const uint32_t*>(tb.lut16k);
    for (int i = t; i < 4096; i += NT) hv::sts_u32(lut + 128u + (uint32_t)(i * 4) + ((uint32_t)(i * 4) & 0x3f80u), hv::ldg(r32 + i));
}

// Store epilogue with the tables in shared memory: same operations, same order as finish_pixel().
//   enc(v)  floatspace_to_srgb (color.rs:59-69): linear -> 16 K table in the LUT holes; sRGB space -> uchar_clamp_ff(255 v)
//   tl(b)   byte_to_float of the working space = the lane's own copy in the replicated LUT
// EPI: 0 = every compositing mode / working space / colour matrix (read from the job); 1 = ReplaceSelf, linear light, no matrix;
// 2 = ReplaceSelf, sRGB space, no matrix (the thumbnail cases: nothing but the encode is compiled).  CH == 4 <=> alpha is meaningful.
template <int EPI, int CH>
__device__ __forceinline__ uint32_t hv_finish_pixel(float b, float g, float r, float a, const uint32_t flags, const JobDev& job,
                                                    const uint32_t lut, const uint32_t lut_lane, const uint8_t* dst) {
    constexpr bool SIMPLE = EPI != 0;
    const bool linear = EPI == 1 ? true : EPI == 2 ? false : (flags & JF_LINEAR) != 0u;
    auto enc = [&](float v) -> uint32_t {
        if (linear) {                                          // lut.rs:4-8
            const float s = __fmul_rn(hv::saturate(v), 16383.0f);   // == min(max(v * 16383, 0), 16383) for every v (lut.rs:4-8): same product inside
                                                                     // [0, 1], the bounds outside, 0 for NaN
            const uint32_t i = (uint32_t)(int)s;
            return hv::lds_lut_u8(lut + 128u + i + (i & 0x3f80u));
        }
        return uchar_clamp_ff(__fmul_rn(255.0f, v));
    };
    constexpr bool am = CH == 4;
    const uint32_t compose = SIMPLE ? 0u : (flags >> JF_COMPOSE_SHIFT) & 3u;
    uint32_t ob, og, orr, oa;
    if (compose == 1u) {                                   // BlendWithSelf: scaling.rs:254-287
        if (a > 0.994f || !am) {
            ob = enc(b); og = enc(g); orr = enc(r); oa = 255u;
        } else {
            const uint32_t d = *reinterpret_cast<const uint32_t*>(dst);
            const float da = (float)(int)(d >> 24);
            const float dc = __fmul_rn(__fsub_rn(1.0f, a), __fadd_rn(__fmul_rn(1.0f / 255.0f, da), 0.0f));
            const float fa = __fadd_rn(a, dc);
            ob = enc(__fdiv_rn(__fadd_rn(b, __fmul_rn(dc, hv::lds_lut(lut_lane + ((d & 0xffu) << 8)))), fa));
            og = enc(__fdiv_rn(__fadd_rn(g, __fmul_rn(dc, hv::lds_lut(lut_lane + (((d >> 8) & 0xffu) << 8)))), fa));
            orr = enc(__fdiv_rn(__fadd_rn(r, __fmul_rn(dc, hv::lds_lut(lut_lane + (((d >> 16) & 0xffu) << 8)))), fa));
            oa = uchar_clamp_ff(__fmul_rn(fa, 255.0f));
        }
    } else if (!am) {                                      // scaling.rs:227-232
        ob = enc(b); og = enc(g); orr = enc(r); oa = 255u;
    } else {
        if (compose == 2u) {                               // BlendWithMatte (scaling.rs:119-148)
            const float t = __fsub_rn(1.0f, a);
            b = __fadd_rn(b, __fmul_rn(t, job.matte[0]));
            g = __fadd_rn(g, __fmul_rn(t, job.matte[1]));
            r = __fadd_rn(r, __fmul_rn(t, job.matte[2]));
            a = __fadd_rn(a, __fmul_rn(t, job.matte[3]));
        }
        if (a > 0.0f) { b = __fdiv_rn(b, a); g = __fdiv_rn(g, a); r = __fdiv_rn(r, a); }
        ob = enc(b); og = enc(g); orr = enc(r);
        oa = uchar_clamp_ff(__fmul_rn(a, 255.0f));
    }
    if (!SIMPLE && (flags & JF_CM)) {                      // color_matrix.rs:5-28, on sRGB bytes
        const float fr = (float)orr, fg = (float)og, fb = (float)ob, fa = (float)oa;
        const float* m = job.cm;
        auto row = [&](int c) {
            float s = __fmul_rn(m[c * 5 + 0], fr);
            s = __fadd_rn(s, __fmul_rn(m[c * 5 + 1], fg));
            s = __fadd_rn(s, __fmul_rn(m[c * 5 + 2], fb));
            s = __fadd_rn(s, __fmul_rn(m[c * 5 + 3], fa));
            return uchar_clamp_ff(__fadd_rn(s, m[c * 5 + 4]));
        };
        orr = row(0); og = row(1); ob = row(2); oa = row(3);
    }
    return ob | (og << 8) | (orr << 16) | (oa << 24);
}

// ORI != HV_ORI_NONE: the resample of orient(in, flag) (ifb200_batch_enqueue_oriented).  The plan is that of the oriented frame, so
// the lanes are oriented rows and the pixel stream runs over oriented columns, as above; only the TMA box and the way a lane reads
// its four pixels of a chunk differ.  A backwards stream axis fetches boxes from the far end and reads chunk 3 - k of a box, its
// four pixels reversed; a backwards lane axis places the box 32 rows (columns) up from the far end and gives lane l box row
// (column) 31 - l.  Transposed (5..8): the box is 32 source columns x 16 source rows, unswizzled; lane l reads word l (or 31 - l)
// of four box rows per chunk, four conflict-free 4-byte loads.  Boxes that reach past the bitmap (negative coordinates included)
// are zero-filled by the TMA unit; their samples carry zero weights.  Box origins along source x stay multiples of four pixels (16
// bytes), as for the stored frame: see the band start below and the engine's choice of jobs for the ring kernel.
// SRC != HV_SRC_BGRA: the resample of to_bgra(rows) (ifb200_batch_enqueue_rows); the plan, the V pass and the store are those of the
// BGRA frame.  RGBA32 reads the BGRA box and swaps blue and red in the look-ups' byte selectors.  RGB24: the tensor is the rows'
// bytes from the 16-byte aligned address at or below `in` (in_xoff = the 0..15 bytes between them, the "phase"), phase + 3 in_w
// bytes wide, zero-filled beyond; the 16 pixels of a box start at byte phase + 3x, so the box origin (phase + 3x) & ~15 stays
// 16-byte aligned and the pixels sit at byte r = (phase + 3x) & 15 of every box row, the same r all along the stream (48 = 0 mod
// 16; r + 48 <= 63).  A lane's chunk k is bytes r + 12k .. r + 12k + 11 of its row: four 4-byte loads (words r/4 + 3k ..) and byte
// permutes give its four pixels as words with red in byte 0, green in byte 1, blue in byte 2 (byte 3 unused: alpha is 255).
// Both together (ifb200_batch_enqueue_rows_oriented): RGBA32 is the BGRA oriented form with the look-ups' blue and red swapped.  RGB24
// flips keep the 64-byte box; a backwards stream axis fetches far-end boxes at byte phase + 3 (W - 16 - x) aligned down to 16, 48
// bytes lower each step, so that r stays constant again, and reads chunk 3 - k, its four pixels reversed; a backwards lane axis gives
// lane l box row 31 - l with that row's swizzle.  RGB24 transposes read boxes of 128 bytes x 16 source rows, unswizzled, whose origin
// is phase + 3 x0 aligned down to 16 (x0: the source column of box column 0; 32 columns are 96 bytes, + up to 15 of r): lane l (or
// 31 - l) finds its pixel at byte r + 3 l of each box row, two 4-byte loads and a byte permute; the 32 lanes' loads fall in 24
// consecutive words.  Byte-aligned origins need neither the band's early start of the BGRA transposes nor a width rule.
// PROF != PF_IDENTITY: the resample of transform_to_srgb(source, profile) (ifb200_batch_enqueue_profiled), every job of the launch
// under one plan, which follows the job array (jobs[n_jobs] as a ProfDev).  The CTA stages its tables next to the flag word (tone
// tables or byte map; the 3 x 3 matrix stays in registers), and conv() runs every source pixel word through pf_step before the
// look-ups, which then see the sRGB bytes the two-step route would have written; its encode reads the linear -> sRGB table in the
// LUT block's holes 0..127.
template <int AV, int CH, int EPI, int ORI = HV_ORI_NONE, int SRC = HV_SRC_BGRA>
__global__ void __launch_bounds__(HvCfg<AV, CH>::kThreads, 1)
hv_ring_kernel(const JobDev* __restrict__ jobs, const HvTmap* __restrict__ tmaps, Tables tb, HvPlanDev pl, uint32_t n_jobs,
               uint32_t* __restrict__ counters) {
    constexpr int PROF = PF_IDENTITY;
#define IFB_HV_PROFILED 0
#include "ifb_hv_ring_body.inc"
#undef IFB_HV_PROFILED
}
template <int AV, int CH, int EPI, int ORI, int SRC, int PROF>
__global__ void __launch_bounds__(HvCfg<AV, CH, PROF>::kThreads, 1)
hv_ring_profiled_kernel(const JobDev* __restrict__ jobs, const HvTmap* __restrict__ tmaps, Tables tb, HvPlanDev pl, uint32_t n_jobs,
                        uint32_t* __restrict__ counters) {
#define IFB_HV_PROFILED 1
#include "ifb_hv_ring_body.inc"
#undef IFB_HV_PROFILED
}
