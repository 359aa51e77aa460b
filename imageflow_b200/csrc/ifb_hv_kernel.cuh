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
    const float* hw;          // [n_strips][hw_stride][AVP]: weight of the open output column in each ring slot, pixel-stream order
    const uint8_t* hdone;     // [n_strips][hw_stride + 64]: output columns completing after this pixel (bits 0..6), V-pass mark (bit 7)
    const float* vw;          // [in_h][AVP]
    const uint8_t* vdone;     // [in_h + 32]
    uint32_t zero;            // 0 (a zero the compiler cannot see: hv::zero_after)
    uint32_t hw_stride;       // source columns (weight records) per strip in hw; hdone has hw_stride + 64 bytes per strip
};
struct alignas(64) HvTmap { unsigned char bytes[128]; };              // CUtensorMap of one job's input bitmap (u32 pixels, box 16 x 32, SWIZZLE_64B)

#ifndef IFB_HV_MAXCOLS4
#define IFB_HV_MAXCOLS4 64             // widest strip of the ring-depth-4 variants (V accumulators: 12 or 16 registers per 16 columns)
#endif
template <int AV, int CH> struct HvCfg {
    static_assert(AV == 4 || AV == 6, "ring depth");
    static constexpr int kAvp = AV == 4 ? 4 : 8;                      // floats per weight record
    static constexpr int kCapPx = 16384 / (kAvp * 4);                 // pixels of H weights that fit in the holes
    static constexpr int kNP = AV / 2;                                // packed slot pairs
    static constexpr int kCG = 32 / kNP;                              // output columns per group: kNP x kCG lanes in the V pass (16, or 10 at ring depth 6)
    static constexpr int kMaxCols = AV == 4 ? IFB_HV_MAXCOLS4 : (CH == 3 ? 50 : 40);   // widest strip (output columns)
    static constexpr int kNG = kMaxCols / kCG + 1;                    // column groups per strip (V accumulators: 2 * CH registers per group); groups end on
                                                                      // chunk-pair boundaries and are not always full, hence one more than the columns need
    static constexpr int kWarps = CH == 3 ? 16 : 12;
    static constexpr int kThreads = kWarps * 32;
    static constexpr int kStages = 2;
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
template <int AV, int CH>
__host__ __device__ constexpr uint32_t hv_layout(uint32_t sb_low16, int warp, uint32_t* st_off, uint32_t* x_off, uint32_t* mb_off) {
    using C = HvCfg<AV, CH>;
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
    return b_mb + W * 8u * (uint32_t)C::kStages + 16u;                // + one CTA-wide flag word (hv_flag_offset)
}
// window offset of the CTA-wide flag word: the last 16 bytes of the layout
template <int AV, int CH> __host__ __device__ constexpr uint32_t hv_flag_offset(uint32_t sb_low16) { return hv_layout<AV, CH>(sb_low16, -1, nullptr, nullptr, nullptr) - 16u; }
template <int AV, int CH> constexpr uint32_t hv_total_bytes(uint32_t sb_low16) { return hv_layout<AV, CH>(sb_low16, -1, nullptr, nullptr, nullptr); }

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

#ifndef IFB_HV_NOFAST
#define IFB_HV_NOFAST 0                // 1: only the general form of a chunk (A/B builds)
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

template <int AV, int CH, int EPI>
__global__ void __launch_bounds__(HvCfg<AV, CH>::kThreads, 1)
hv_ring_kernel(const JobDev* __restrict__ jobs, const HvTmap* __restrict__ tmaps, Tables tb, HvPlanDev pl, uint32_t n_jobs,
               uint32_t* __restrict__ counters) {
    using C = HvCfg<AV, CH>;
    constexpr int AVP = C::kAvp, NG = C::kNG, NP = C::kNP, S = C::kStages, CG = C::kCG;
    constexpr uint32_t kRec = (uint32_t)AVP * 4u;                          // bytes per H weight record (one source column)
    constexpr uint32_t kXCol = (uint32_t)C::kXPitch * 4u;                  // bytes per column of the exchange buffer
    IFB_HV_DYNAMIC_SMEM(hv_smem);
    const uint32_t sb = hv::smem_u32(hv_smem);
    const uint32_t lut = sb + ((0x10000u - (sb & 0xffffu)) & 0xffffu);     // window address of the LUT block: low 16 bits are zero
    const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
    // A value that is the same in every lane, rebuilt from a warp vote: the compiler then KNOWS it is warp-uniform.
    auto uni = [&](uint32_t v) -> uint32_t { return hv::ballot((v >> lane) & 1u); };
    uint32_t stb, xbuf, mb;                                                // this warp's stage ring, exchange buffer, mbarriers (window addresses)
    {
        uint32_t o_st = 0, o_x = 0, o_mb = 0;
        hv_layout<AV, CH>(sb & 0xffffu, warp, &o_st, &o_x, &o_mb);
        stb = sb + o_st; xbuf = sb + o_x; mb = sb + o_mb;
    }
    const uint32_t flagw = sb + hv_flag_offset<AV, CH>(sb & 0xffffu);
    const uint32_t flags0 = jobs[0].flags;                                 // working space and channel count are the same for all jobs of a launch

    hv_fill_luts<C::kThreads>(lut, tb, flags0, t);
    if (lane == 0) {
        for (int s = 0; s < S; ++s) hv::mbar_init(mb + 8u * s, 1u);
        hv::mbar_init_fence();
    }
    uint32_t par = 0;                                                      // bit s: parity the next wait on stage s expects

    const uint32_t lut_lane = lut + (uint32_t)lane * 4u;
    const uint32_t lane4 = ((uint32_t)lane * 4u) | ((lut >> 16) << 8);     // PRMT operand: byte 0 = lane*4, bytes 1..2 = window bits 16..31
    // SWIZZLE_64B: 16-byte chunk index ^= (address >> 7) & 3; this lane's row starts at lane * 64: chunk k of "my row" lies at
    // lane * 64 + ((k << 4) ^ swz)
    const uint32_t swz = (((uint32_t)lane >> 1) & 3u) << 4;
    const uint32_t n_bands = (uint32_t)pl.n_bands;
    const uint32_t n_items = n_jobs * n_bands;
    const uint32_t lutw = lut + 128u * 256u + 128u;                        // hole 128: the strip's H weights
    const bool leader = hv::elect_one();                                   // the lane that talks to the TMA unit
    // V pass role of this lane: slot pair vh (ring slots 2 vh, 2 vh + 1) of column cl of the group; lanes beyond NP * CG idle
    const uint32_t vh = (uint32_t)lane / (uint32_t)CG, cl = (uint32_t)lane % (uint32_t)CG;
    const bool vlane = vh < (uint32_t)NP;
    const uint32_t xr = xbuf + cl * kXCol;
    const uint32_t xw0 = xbuf + (uint32_t)lane * 4u;                       // H pass role: row `lane` of column 0

    for (int sv = 0; sv < pl.n_strips; ++sv) {
        // The next strip (from this CTA's starting strip on) whose work counter has not run out: warp 0 looks at up to 32 counters
        // at once.  A launch for one small image has more strips than items per CTA, and every CTA used to copy every strip's
        // weight table whether or not anything was left to do there (most of the 70 us such a launch took).
        if (warp == 0) {
            const int k = sv + lane;
            const bool work = k < pl.n_strips && hv::ldg_volatile(counters + (blockIdx.x + (uint32_t)k) % (uint32_t)pl.n_strips) < n_items;
            const uint32_t m = hv::ballot(work);
            if (lane == 0) hv::sts_u32(flagw, m ? (uint32_t)__ffs((int)m) : (sv + 32 < pl.n_strips ? 33u : 0u));
        }
        hv::cta_sync();                                                    // every warp is done with the previous strip's weights (first time: tables filled)
        const uint32_t skip1 = hv::lds_u32(flagw);                         // 0: nothing left anywhere; 1..32: strips to skip + 1; 33: none of these 32
        hv::cta_sync();                                                    // (the flag word is rewritten by the next look)
        if (skip1 == 0u) break;
        if (skip1 == 33u) { sv += 31; continue; }
        sv += (int)skip1 - 1;
        const int s = (int)((blockIdx.x + (uint32_t)sv) % (uint32_t)pl.n_strips);
        const HvStripDev sd_ = pl.strips[s];
        const int sX0 = (int)uni((uint32_t)sd_.X0);
        const uint32_t sH0 = uni((uint32_t)sd_.hslot0);
        const int sK0 = (int)uni((uint32_t)sd_.k0), nst = (int)uni((uint32_t)sd_.nst);
        {   // H weights of the strip: 16-byte units u -> hole 128 + u/8, offset (u%8)*16
            const float4* __restrict__ src = reinterpret_cast<const float4*>(pl.hw + (size_t)s * pl.hw_stride * AVP);
            const int n16 = (nst * 16 + 4) * AVP / 4;                      // + one chunk: the pipeline fetches one record ahead
            for (int u = t; u < n16; u += C::kThreads) hv::sts_f32x4(lutw + ((uint32_t)(u >> 3) << 8) + ((uint32_t)(u & 7) << 4), hv::ldg(src + u));
        }
        hv::cta_sync();
        const uint8_t* __restrict__ hdone = pl.hdone + (size_t)s * (pl.hw_stride + 64u);
        const uint32_t npairs = (uint32_t)nst * 2u;                        // chunk pairs (eight source columns) per row block

        for (;;) {
            uint32_t item = 0;
            if (lane == 0) item = hv::atomic_inc(counters + s);
            item = uni(hv::bcast0(item));
            if (item >= n_items) break;
            const uint32_t job_i = item / n_bands, band_i = item - job_i * n_bands;
            const JobDev& job = jobs[job_i];
            const HvTmap* tm = tmaps + job_i;
            const HvBandDev bd_ = pl.bands[band_i];
            const int bJ0 = (int)uni((uint32_t)bd_.j0), bNr = (int)uni((uint32_t)bd_.nrows);
            const int bY0 = (int)uni((uint32_t)bd_.Y0), bY1 = (int)uni((uint32_t)bd_.Y1);
            const uint32_t flags = uni(job.flags);
            const int nrb = (bNr + 31) >> 5;
            const int x_origin = sK0 + (int)uni(job.in_xoff);

            // ---- TMA pipeline state: boxes are fetched row block by row block, left to right
            const int x_end = x_origin + nst * 16;
            int tma_x = x_origin, tma_y = bJ0, tma_left = nrb * nst, is_s = 0;   // next box to fetch, boxes not fetched yet, the ring slot it goes to
            auto issue = [&](const uint32_t zero_dep) {                    // zero_dep: 0, computed from what the slot's last load returned
                hv::warp_sync();                                           // every lane has read what the refilled slot held
                if (leader) {
                    const uint32_t bar = mb + 8u * (uint32_t)is_s;
                    hv::mbar_expect_tx(bar, (uint32_t)C::kStageBytes);
                    hv::tma_load_box(stb + (uint32_t)is_s * C::kStageBytes, tm, tma_x + (int)zero_dep, tma_y, bar);
                }
                --tma_left; is_s ^= 1;
                tma_x += 16;
                if (tma_x == x_end) { tma_x = x_origin; tma_y += 32; }
            };
            static_assert(S == 2, "the slot bookkeeping below toggles between two slots");
            if (tma_left > 0) issue(0u);
            int cs_s = 0;                                                  // ring slot of the stage being consumed

            float2 accV[NG][CH];                                           // this lane's slot pair of column cl of every group
#pragma unroll
            for (int gq = 0; gq < NG; ++gq)
#pragma unroll
                for (int c = 0; c < CH; ++c) accV[gq][c] = make_float2(0.0f, 0.0f);
            int Yc = (int)uni((uint32_t)bd_.Yf);                           // next output row to complete at the start of the row block, and its slot
            uint32_t vslot = uni((uint32_t)bd_.vslot0);
            uint8_t* const out_col = job.out + (size_t)(sX0 + (int)cl) * 4;
            const size_t out_stride = job.out_stride;

            for (int rb = 0; rb < nrb; ++rb) {
                const int row0 = bJ0 + rb * 32;
                uint32_t vm1, vm2, vtot;                                   // rows of the block completing output rows
                {
                    const uint32_t vd = lane < bNr - rb * 32 ? (uint32_t)hv::ldg(pl.vdone + row0 + lane) : 0u;
                    vm1 = hv::ballot(vd >= 1u); vm2 = hv::ballot(vd >= 2u); vtot = hv::warp_sum(vd);
                }
                float2 accH[CH][NP];
#pragma unroll
                for (int c = 0; c < CH; ++c)
#pragma unroll
                    for (int q = 0; q < NP; ++q) accH[c][q] = make_float2(0.0f, 0.0f);
                uint32_t hslot = sH0, colbuf = 0, grp = 0, gX = 0;         // ring slot of the next column to complete; columns parked since the last V pass; group; its first column
                uint32_t xw = xw0;                                         // where this lane parks its value of the next completed column
                uint32_t wcur = lutw;                                      // H weight records of the current chunk pair

                // ---- first stage of the row block
                if (tma_left > 0) issue(0u);
                hv::mbar_wait(mb + 8u * (uint32_t)cs_s, (par >> cs_s) & 1u);
                par ^= 1u << cs_s;
                uint32_t sbase = stb + (uint32_t)cs_s * C::kStageBytes + (uint32_t)lane * 64u;
                uint4 rawA = hv::lds_u32x4(sbase + swz), rawB;             // the sixteen bytes of this lane's row in the pair's first / second chunk
                uint32_t hd_next = (uint32_t)hv::ldg(hdone + lane);
                uint32_t HM1 = 0, HM2 = 0, HMV = 0;

                // The pixel loop is software-pipelined by one source column: while column i is multiply-added, column i+1 is being
                // converted (its table look-ups are in flight) and its weight record fetched.
                float P0[CH], P1[CH];
                float2 W0[NP], W1[NP];
                auto conv = [&](float (&P)[CH], const uint32_t v) {
                    P[0] = hv::lut_gather<0x6504>(v, lane4); P[1] = hv::lut_gather<0x6514>(v, lane4); P[2] = hv::lut_gather<0x6524>(v, lane4);
                    if (CH == 4) {                                         // alpha table entry == a * (1/255f) (color.rs:38): computed, not gathered
                        const float af = __fmul_rn(__uint2float_rn(v >> 24), 1.0f / 255.0f);
                        P[0] = __fmul_rn(P[0], af); P[1] = __fmul_rn(P[1], af); P[2] = __fmul_rn(P[2], af); P[CH - 1] = af;
                    }
                };
                auto wload = [&](float2 (&W)[NP], const uint32_t a) {
                    const float4 q4 = hv::lds_w4(a);
                    W[0] = make_float2(q4.x, q4.y); W[1] = make_float2(q4.z, q4.w);
                    if (AV == 6) W[NP - 1] = hv::lds_w2(a + 16u);
                };
                auto mac = [&](const float (&P)[CH], const float2 (&W)[NP]) {
#pragma unroll
                    for (int c = 0; c < CH; ++c) {
                        const float2 v_ = make_float2(P[c], P[c]);
#pragma unroll
                        for (int q = 0; q < NP; ++q) accH[c][q] = hv::ffma2(W[q], v_, accH[c][q]);
                    }
                };
                wload(W0, wcur); conv(P0, rawA.x);

                // The loop body is a PAIR of chunks (eight source columns): per-chunk bookkeeping is paid once for two, and the V pass
                // marks sit on pair ends.
                for (uint32_t pq = 0; pq < npairs; pq += 4u) {
                    // completion masks of the next 32 source columns (four pairs); the bytes after them are on their way
                    HM1 = hv::ballot((hd_next & 0x7fu) >= 1u); HM2 = hv::ballot((hd_next & 0x7fu) >= 2u); HMV = hv::ballot((hd_next & 0x80u) != 0u);
                    hd_next = (uint32_t)hv::ldg(hdone + (pq + 4u) * 8u + (uint32_t)lane);
                    const uint32_t pe = min(pq + 4u, npairs);
#pragma unroll 1
                  for (uint32_t pc = pq; pc < pe; ++pc) {
                    const uint32_t hm = HM1, hm2 = HM2, hmv = HMV;
                    HM1 >>= 8; HM2 >>= 8; HMV >>= 8;
                    const uint32_t wB = wcur + (AV == 4 ? 64u : 256u);     // second chunk's records
                    const uint32_t wnext = wcur + (AV == 4 ? 256u : 512u); // next pair's
                    const bool more = pc + 1u < npairs;

                    // a completed output column: its CH values are parked in the exchange buffer, the ring slot is cleared
#define IFB_HV_SLOT(S_) case S_: if (S_ < AV) { _Pragma("unroll") for (int ch_ = 0; ch_ < CH; ++ch_) { \
        float& a_ = (S_ & 1) ? accH[ch_][(S_ % AV) / 2].y : accH[ch_][(S_ % AV) / 2].x; \
        hv::sts_f32(xw + (uint32_t)ch_ * 128u, a_); a_ = 0.0f; } } break;
#define IFB_HV_FLUSH(I_) if ((hm >> (I_)) & 1u) { \
        uint32_t n_ = 1u; \
        if ((hm2 >> (I_)) & 1u) n_ = uni((uint32_t)hv::ldg(hdone + pc * 8u + (I_)) & 0x7fu); \
        _Pragma("unroll 1") do { \
            switch (hslot) { IFB_HV_SLOT(0) IFB_HV_SLOT(1) IFB_HV_SLOT(2) IFB_HV_SLOT(3) IFB_HV_SLOT(4) IFB_HV_SLOT(5) default: break; } \
            xw += kXCol; ++colbuf; hslot = hslot + 1u == (uint32_t)AV ? 0u : hslot + 1u; \
        } while (--n_); }

                    // Second chunk's bytes (chunk 2 pc + 1, same stage as the first).  With them in registers the second pair of a stage has
                    // read its stage completely: the slot is refilled and the next stage waited for before the pair starts (the refill is
                    // made to depend on the loaded bytes, so that it cannot overtake the load).
                    rawB = hv::lds_u32x4(sbase + (((((pc & 1u) << 1) | 1u) << 4) ^ swz));
                    if ((pc & 1u) && more) {
                        cs_s ^= 1;
                        if (tma_left > 0) issue(hv::zero_after(rawB.x, pl.zero));
                        hv::mbar_wait(mb + 8u * (uint32_t)cs_s, (par >> cs_s) & 1u);
                        par ^= 1u << cs_s;
                        sbase = stb + (uint32_t)cs_s * C::kStageBytes + (uint32_t)lane * 64u;
                    }
                    // behind the pair's seventh column: the next pair's first chunk (chunk 2 pc + 2; behind the last pair of the row block: bytes nobody uses)
#define IFB_HV_RELOAD rawA = hv::lds_u32x4(sbase + (((((pc + 1u) & 1u) << 1) << 4) ^ swz));
                    // A chunk (four source columns) exists in six compiled forms, picked by tests whose operands are known long before
                    // they are needed: no completion (plain straight-line code: about half of the chunks of a 7.5 : 1 down-scale); exactly
                    // one completion and no column that completes twice -- one form per ring slot of the completing column, with a
                    // predicated "park and clear" of that slot behind every column (no branch inside, no look-up of the slot); and
                    // the general form with a test behind every column.
#define IFB_HV_ACC(S_, C_) (((S_) & 1) ? accH[C_][((S_) % AV) / 2].y : accH[C_][((S_) % AV) / 2].x)
#define IFB_HV_PF(S_, BIT_, M_) { \
        if (CH == 3) hv::flush3_if<BIT_, kXCol>(xw, IFB_HV_ACC(S_, 0), IFB_HV_ACC(S_, 1), IFB_HV_ACC(S_, 2), M_); \
        else hv::flush4_if<BIT_, kXCol>(xw, IFB_HV_ACC(S_, 0), IFB_HV_ACC(S_, 1), IFB_HV_ACC(S_, 2), IFB_HV_ACC(S_, CH - 1), M_); }
#define IFB_HV_NONE
#define IFB_HV_STEPS_A(F0_, F1_, F2_, F3_) { \
        wload(W1, wcur + kRec); conv(P1, rawA.y); mac(P0, W0); F0_ \
        wload(W0, wcur + 2u * kRec); conv(P0, rawA.z); mac(P1, W1); F1_ \
        wload(W1, wcur + 3u * kRec); conv(P1, rawA.w); mac(P0, W0); F2_ \
        wload(W0, wB); conv(P0, rawB.x); mac(P1, W1); F3_ }
#define IFB_HV_STEPS_B(F0_, F1_, F2_, F3_) { \
        wload(W1, wB + kRec); conv(P1, rawB.y); mac(P0, W0); F0_ \
        wload(W0, wB + 2u * kRec); conv(P0, rawB.z); mac(P1, W1); F1_ \
        wload(W1, wB + 3u * kRec); conv(P1, rawB.w); IFB_HV_RELOAD mac(P0, W0); F2_ \
        wload(W0, wnext); conv(P0, rawA.x); mac(P1, W1); F3_ }
#define IFB_HV_CHUNK(STEPS_, SH_) { \
        const uint32_t m4_ = (hm >> (SH_)) & 15u; \
        if (IFB_HV_NOFAST || ((((hm2 >> (SH_)) & 15u) | (m4_ & (m4_ - 1u))) != 0u)) { \
            STEPS_(IFB_HV_FLUSH((SH_) + 0), IFB_HV_FLUSH((SH_) + 1), IFB_HV_FLUSH((SH_) + 2), IFB_HV_FLUSH((SH_) + 3)) \
        } else if (m4_ == 0u) { \
            STEPS_(IFB_HV_NONE, IFB_HV_NONE, IFB_HV_NONE, IFB_HV_NONE) \
        } else { \
            if (hslot < 2u) { \
                if (hslot == 0u) IFB_HV_FORM(STEPS_, 0) else IFB_HV_FORM(STEPS_, 1) \
            } else if (AV == 4 || hslot < 4u) { \
                if (hslot == 2u) IFB_HV_FORM(STEPS_, 2) else IFB_HV_FORM(STEPS_, 3) \
            } else { \
                if (hslot == 4u) IFB_HV_FORM(STEPS_, 4) else IFB_HV_FORM(STEPS_, 5) \
            } \
            ++colbuf; hslot = hslot + 1u == (uint32_t)AV ? 0u : hslot + 1u; \
        } }
#define IFB_HV_FORM(STEPS_, K_) STEPS_(IFB_HV_PF((K_) % AV, 1u, m4_), IFB_HV_PF((K_) % AV, 2u, m4_), IFB_HV_PF((K_) % AV, 4u, m4_), IFB_HV_PF((K_) % AV, 8u, m4_))
                    IFB_HV_CHUNK(IFB_HV_STEPS_A, 0)
                    IFB_HV_CHUNK(IFB_HV_STEPS_B, 4)
#undef IFB_HV_CHUNK
#undef IFB_HV_FORM
#undef IFB_HV_STEPS_A
#undef IFB_HV_STEPS_B
#undef IFB_HV_NONE
#undef IFB_HV_PF
#undef IFB_HV_ACC
#undef IFB_HV_RELOAD
#undef IFB_HV_FLUSH
#undef IFB_HV_SLOT
                    wcur = wnext;

                    if ((hmv >> 7) & 1u) {
                        // ---- V pass of the columns parked since the last one (a "group", at most CG of them; the host put the mark where the
                        // group is full or the strip ends): lane = (slot pair vh, output column sX0 + gX + cl).  The 32 H-filtered rows of the
                        // block are multiply-added, in row order, into the lane's pair of vertical accumulators (output row Y owns slot Y mod AV);
                        // a completed output row goes through the store epilogue in the lanes whose pair holds its slot.
                        hv::warp_sync();
                        const bool col_live = vlane && cl < colbuf;
                        uint8_t* const out_px = out_col + (size_t)gX * 4;
                        // the group's accumulators: fetched from / returned to the register set of group `grp` by two small switches, so that
                        // the V pass code exists once
                        float2 acc[CH];
                        switch (grp) {
#define IFB_HV_VGROUP(G_) case G_: if (G_ < NG) { _Pragma("unroll") for (int ch_ = 0; ch_ < CH; ++ch_) acc[ch_] = accV[(G_) % NG][ch_]; } break;
                        IFB_HV_VGROUP(0) IFB_HV_VGROUP(1) IFB_HV_VGROUP(2) IFB_HV_VGROUP(3) IFB_HV_VGROUP(4) IFB_HV_VGROUP(5) IFB_HV_VGROUP(6) IFB_HV_VGROUP(7) IFB_HV_VGROUP(8)
#undef IFB_HV_VGROUP
                        default:
#pragma unroll
                            for (int ch_ = 0; ch_ < CH; ++ch_) acc[ch_] = make_float2(0.0f, 0.0f);
                            break;
                        }
                        {
                            // Completed output rows are not encoded where they complete: the lanes that hold the row's slot park its values in
                            // the exchange buffer -- row k of their column for the k-th completion of the block; rows 0..k of the buffer have
                            // been consumed by then -- and the store epilogue runs afterwards over the parked rows with ALL lanes at work
                            // (lane = (row k mod NP, column)) and no branch in its body.
                            int Yb = Yc;                                   // output row of parked row 0
                            uint32_t nc = 0;                               // rows parked
                            uint32_t vs = vslot;
                            auto drain = [&]() {
                                hv::warp_sync();
#pragma unroll 1
                                for (uint32_t k0 = 0; k0 < nc; k0 += (uint32_t)NP) {
                                    const uint32_t k = k0 + (vlane ? vh : 0u);
                                    float f_[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
                                    for (int ch_ = 0; ch_ < CH; ++ch_) f_[ch_] = hv::lds_f32(xr + (uint32_t)ch_ * 128u + (k & 31u) * 4u);
                                    const int Yl = Yb + (int)k;
                                    const bool mine = k < nc && Yl >= bY0 && Yl < bY1 && col_live;
                                    uint8_t* dst = out_px + (size_t)Yl * out_stride;
                                    if (EPI != 0) {                        // the encode never reads the canvas: every lane runs it, the owners store
                                        const uint32_t px_ = hv_finish_pixel<EPI, CH>(f_[0], f_[1], f_[2], CH == 4 ? f_[3] : 0.0f, flags, job, lut, lut_lane, dst);
                                        if (mine) *reinterpret_cast<uint32_t*>(dst) = px_;
                                    } else if (mine) {
                                        *reinterpret_cast<uint32_t*>(dst) = hv_finish_pixel<EPI, CH>(f_[0], f_[1], f_[2], CH == 4 ? f_[3] : 0.0f, flags, job, lut, lut_lane, dst);
                                    }
                                }
                                hv::warp_sync();
                                Yb += (int)nc; nc = 0;
                            };
                            const float* __restrict__ vwp = pl.vw + (size_t)row0 * AVP + 2u * (vlane ? vh : 0u);   // this lane's pair of V weights, row by row
                            uint32_t xrr = xr;
                            auto vrow = [&](const float* __restrict__ wp, const uint32_t xa_) {
                                const float2 wv = hv::ldg(reinterpret_cast<const float2*>(wp));
#pragma unroll
                                for (int ch_ = 0; ch_ < CH; ++ch_) {
                                    const float x_ = hv::lds_f32(xa_ + (uint32_t)ch_ * 128u);
                                    acc[ch_] = hv::ffma2(wv, make_float2(x_, x_), acc[ch_]);
                                }
                            };
                            auto vrow2 = [&](const float* __restrict__ wp, const uint32_t xa_) {      // rows r, r + 1 (r even): one 8-byte access per channel
                                const float2 wa = hv::ldg(reinterpret_cast<const float2*>(wp)), wb = hv::ldg(reinterpret_cast<const float2*>(wp + AVP));
#pragma unroll
                                for (int ch_ = 0; ch_ < CH; ++ch_) {
                                    const float2 x_ = hv::lds_w2(xa_ + (uint32_t)ch_ * 128u);
                                    acc[ch_] = hv::ffma2(wa, make_float2(x_.x, x_.x), acc[ch_]);
                                    acc[ch_] = hv::ffma2(wb, make_float2(x_.y, x_.y), acc[ch_]);
                                }
                            };
                            // all 32 rows of the block (rows below the band's last carry no completion bit, and what they add to a slot is never
                            // read), in runs that end with a row that completes an output row; a run is walked two rows at a time from its
                            // first even row
                            for (int r = 0; r < 32;) {
                                const uint32_t rest = vm1 >> r;
                                int n = rest ? __ffs((int)rest) : 32 - r;
                                r += n;
                                if (((xrr - xr) & 4u) != 0u) { vrow(vwp, xrr); vwp += AVP; xrr += 4u; --n; }
#pragma unroll 1
                                for (int i = n >> 1; i > 0; --i, vwp += 2 * AVP, xrr += 8u) vrow2(vwp, xrr);
                                if (n & 1) { vrow(vwp, xrr); vwp += AVP; xrr += 4u; }
                                if (rest != 0u) {
                                    uint32_t nv = 1u;
                                    if (vm2 != 0u && ((vm2 >> (r - 1)) & 1u)) nv = uni((uint32_t)hv::ldg(pl.vdone + row0 + r - 1));
#pragma unroll 1
                                    for (uint32_t e2 = 0; e2 < nv; ++e2) {
                                        if (nc >= (uint32_t)r) drain();    // (only when several rows complete at once near the top of a block)
                                        hv::warp_sync();                   // the column's other lanes have read the row that is about to be overwritten
                                        const bool holder = (vs >> 1) == vh;
                                        const uint32_t pa = xr + nc * 4u;
                                        if (vs & 1u) {
#pragma unroll
                                            for (int ch_ = 0; ch_ < CH; ++ch_) if (holder) { hv::sts_f32(pa + (uint32_t)ch_ * 128u, acc[ch_].y); acc[ch_].y = 0.0f; }
                                        } else {
#pragma unroll
                                            for (int ch_ = 0; ch_ < CH; ++ch_) if (holder) { hv::sts_f32(pa + (uint32_t)ch_ * 128u, acc[ch_].x); acc[ch_].x = 0.0f; }
                                        }
                                        ++nc; vs = vs + 1u == (uint32_t)AV ? 0u : vs + 1u;
                                    }
                                }
                            }
                            drain();
                        }
                        switch (grp) {
#define IFB_HV_VGROUP(G_) case G_: if (G_ < NG) { _Pragma("unroll") for (int ch_ = 0; ch_ < CH; ++ch_) accV[(G_) % NG][ch_] = acc[ch_]; } break;
                        IFB_HV_VGROUP(0) IFB_HV_VGROUP(1) IFB_HV_VGROUP(2) IFB_HV_VGROUP(3) IFB_HV_VGROUP(4) IFB_HV_VGROUP(5) IFB_HV_VGROUP(6) IFB_HV_VGROUP(7) IFB_HV_VGROUP(8)
#undef IFB_HV_VGROUP
                        default: break;
                        }
                        hv::warp_sync();
                        ++grp; gX += colbuf; colbuf = 0; xw = xw0;
                    }
                  }
                }
                cs_s ^= 1;
                // every group of the row block has seen the same rows: commit the vertical position
                Yc += (int)vtot;
                vslot = (vslot + vtot) % (uint32_t)AV;
            }
        }
    }
}
