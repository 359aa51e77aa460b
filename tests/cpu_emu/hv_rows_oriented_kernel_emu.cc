// Runs the ORIENTED ROW-FORMAT forms of imageflow_b200/csrc/ifb_hv_kernel.cuh -- hv_ring_kernel<AV, CH, EPI, ORI, SRC> with ORI =
// HV_ORI_FLIP / HV_ORI_TRANSPOSE and SRC = HV_SRC_RGBA / HV_SRC_RGB24, the product's CUDA source unmodified -- on the CPU, the way
// hv_rows_kernel_emu.cc and hv_oriented_kernel_emu.cc run the row and the oriented forms: one OS thread per CUDA thread of a CTA, a
// per-warp std::barrier behind every warp-synchronous primitive, shared memory as an exactly-sized heap block addressed through fake
// "shared window" addresses.  The TMA box load is emulated for all four tensor maps of these forms: u32 elements in boxes of 16 x 32
// (SWIZZLE_64B) and 32 x 16 (no swizzle), u8 elements in boxes of 64 bytes x 32 rows (SWIZZLE_64B) and 128 bytes x 16 rows (no
// swizzle); zero fill outside the tensor (past phase + 3 in_w bytes of a row, and at negative coordinates).  A box reads the tensor's
// rows only (stride apart, w elements each).  Every box origin along x is checked to be 16 bytes from the tensor map's 16-byte
// aligned base.  The mbarrier phases are checked.  CTAs of the grid run one after the other.  Built with -ffp-contract=off; with
// -fsanitize=address a run is also a memory check of the kernel.
// TEST INFRASTRUCTURE: nothing in the product calls this; the GPU remains the place where the kernel is run and timed.
#include "cuda_emu.h"

#include <atomic>
#include <barrier>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <thread>
#include <vector>

#define IFB_HV_EMU 1
namespace emu {
static unsigned char* smem;
static size_t smem_bytes;
static uint32_t win_base;                                  // fake shared-window address of smem[0]
static std::barrier<>* block_barrier;
static std::barrier<>* warp_barrier[16];
static uint32_t warp_scratch[16][32];
static std::atomic<int> bad_access{0};
static inline unsigned char* at(uint32_t a, size_t n) {
    const uint64_t off = (uint64_t)a - win_base;
    if (a < win_base || off + n > smem_bytes) { bad_access++; static unsigned char dummy[64]; return dummy; }
    return smem + off;
}
}  // namespace emu

// w: elements per row (u32 pixels, or bytes when `bytes`); `transposed`: the box shape of flags 5..8; same size as a CUtensorMap
struct EmuTmap { const uint8_t* base; uint32_t w, h, stride, bytes, transposed; unsigned char pad[128 - 8 - 20]; };

namespace hv {
static inline unsigned wid() { return threadIdx.x >> 5; }
static inline unsigned lid() { return threadIdx.x & 31; }
static inline void wbar() { emu::warp_barrier[wid()]->arrive_and_wait(); }
static inline uint32_t smem_u32(const void* p) { return (uint32_t)((const unsigned char*)p - emu::smem) + emu::win_base; }
template <class T> static inline T ld(uint32_t a) { T v; std::memcpy(&v, emu::at(a, sizeof(T)), sizeof(T)); return v; }
template <class T> static inline void st(uint32_t a, T v) { std::memcpy(emu::at(a, sizeof(T)), &v, sizeof(T)); }
static inline float lds_lut(uint32_t a) { return ld<float>(a); }
static inline uint32_t lds_lut_u8(uint32_t a) { return ld<uint8_t>(a); }
static inline float4 lds_w4(uint32_t a) { if (a & 15) emu::bad_access++; return ld<float4>(a); }
static inline float2 lds_w2(uint32_t a) { if (a & 7) emu::bad_access++; return ld<float2>(a); }
static inline float lds_f32(uint32_t a) { return ld<float>(a); }
static inline uint4 lds_u32x4(uint32_t a) { if (a & 15) emu::bad_access++; return ld<uint4>(a); }
static inline void sts_f32(uint32_t a, float v) { st(a, v); }
static inline void sts_u32(uint32_t a, uint32_t v) { st(a, v); }
static inline void sts_f32x4(uint32_t a, float4 v) { if (a & 15) emu::bad_access++; st(a, v); }
template <uint32_t BIT, uint32_t STEP> static inline void flush3_if(uint32_t& xw, float& a0, float& a1, float& a2, uint32_t mask) {
    if (mask & BIT) { sts_f32(xw, a0); sts_f32(xw + 128u, a1); sts_f32(xw + 256u, a2); a0 = a1 = a2 = 0.0f; xw += STEP; }
}
template <uint32_t BIT, uint32_t STEP> static inline void flush4_if(uint32_t& xw, float& a0, float& a1, float& a2, float& a3, uint32_t mask) {
    if (mask & BIT) { sts_f32(xw, a0); sts_f32(xw + 128u, a1); sts_f32(xw + 256u, a2); sts_f32(xw + 384u, a3); a0 = a1 = a2 = a3 = 0.0f; xw += STEP; }
}
static inline uint32_t zero_after(uint32_t v, uint32_t zero) { return v & zero; }
static inline float saturate(float v) { return v != v ? 0.0f : (v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v)); }
static inline uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
    const uint64_t src = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; ++i) r |= (uint32_t)((src >> (8 * ((sel >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
}
template <uint32_t SEL> static inline float lut_gather(uint32_t px, uint32_t lane4) { return lds_lut(prmt(px, lane4, SEL)); }
static inline float2 ffma2(float2 a, float2 b, float2 c) { return float2{std::fmaf(a.x, b.x, c.x), std::fmaf(a.y, b.y, c.y)}; }
static inline uint32_t ballot(bool p) {
    emu::warp_scratch[wid()][lid()] = p ? 1u : 0u;
    wbar();
    uint32_t m = 0;
    for (int i = 0; i < 32; ++i) m |= emu::warp_scratch[wid()][i] << i;
    wbar();
    return m;
}
static inline uint32_t bcast0(uint32_t v) {
    if (lid() == 0) emu::warp_scratch[wid()][0] = v;
    wbar();
    const uint32_t r = emu::warp_scratch[wid()][0];
    wbar();
    return r;
}
static inline uint32_t warp_sum(uint32_t v) {
    emu::warp_scratch[wid()][lid()] = v;
    wbar();
    uint32_t s = 0;
    for (int i = 0; i < 32; ++i) s += emu::warp_scratch[wid()][i];
    wbar();
    return s;
}
static inline void warp_sync() { wbar(); }
static inline bool elect_one() { return lid() == 0; }
static inline void cta_sync() { emu::block_barrier->arrive_and_wait(); }
static inline uint32_t atomic_inc(uint32_t* p) { return __atomic_fetch_add(p, 1u, __ATOMIC_SEQ_CST); }
// mbarrier: the issuing lane copies synchronously, so a wait only has to order the warp behind its own lane 0; the phase
// bookkeeping of the kernel is checked nevertheless (expect_tx / complete / parity).
struct Mbar { uint32_t phase; uint32_t pending; };
static inline void mbar_init(uint32_t addr, uint32_t) { st(addr, Mbar{0u, 0u}); }
static inline void mbar_init_fence() {}
static inline void mbar_expect_tx(uint32_t addr, uint32_t bytes) { Mbar m = ld<Mbar>(addr); if (m.pending) emu::bad_access++; m.pending = bytes; st(addr, m); }
static inline void mbar_wait(uint32_t addr, uint32_t parity) {
    wbar();
    const Mbar m = ld<Mbar>(addr);
    if (m.pending != 0 || ((m.phase & 1u) == parity)) emu::bad_access++;      // the phase with this parity must have completed
    wbar();
}
// One box: 32 rows x 64 bytes -- u8 elements x .. x + 63 or u32 elements x .. x + 15 of rows y .. y + 31, row r at dst + 64 r, its
// 16-byte unit c at ((c ^ (row address >> 7) & 3) << 4): SWIZZLE_64B -- or, transposed, 16 rows x 128 bytes -- u8 elements x .. x +
// 127 or u32 elements x .. x + 31 of rows y .. y + 15, row r at dst + 128 r, unswizzled.
static inline void tma_load_box(uint32_t dst, const void* tmv, int x, int y, uint32_t mbar) {
    const EmuTmap* tm = static_cast<const EmuTmap*>(tmv);
    const int esz = tm->bytes ? 1 : 4;
    const int rows = tm->transposed ? 16 : 32, rb = tm->transposed ? 128 : 64;
    if (dst & 127) emu::bad_access++;
    if (((int64_t)x * esz) & 15) emu::bad_access++;                  // box origins stay 16-byte aligned
    for (int r = 0; r < rows; ++r) {
        const int64_t yy = (int64_t)y + r;
        uint8_t row[128];
        for (int i = 0; i < rb; ++i) {
            const int64_t e = (int64_t)x + i / esz;                   // element of the byte
            row[i] = (e >= 0 && yy >= 0 && e < tm->w && yy < tm->h) ? tm->base[(size_t)yy * tm->stride + (size_t)e * esz + (size_t)(i % esz)] : 0;
        }
        const uint32_t ra = dst + (uint32_t)(r * rb);
        if (tm->transposed) std::memcpy(emu::at(ra, 128), row, 128);
        else for (uint32_t c = 0; c < 4; ++c) std::memcpy(emu::at(ra + ((c ^ ((ra >> 7) & 3u)) << 4), 16), row + c * 16, 16);
    }
    Mbar m = ld<Mbar>(mbar);
    if (m.pending < 2048u) emu::bad_access++;
    m.pending -= 2048u;
    if (m.pending == 0u) m.phase ^= 1u;
    st(mbar, m);
}
static inline void tma_prefetch_box(const void*, int, int) {}
template <class T> static inline T ldg(const T* p) { return *p; }
static inline uint32_t ldg_volatile(const uint32_t* p) { return __atomic_load_n(p, __ATOMIC_SEQ_CST); }
static inline uint32_t lds_u32(uint32_t a) { if (a & 3) emu::bad_access++; return ld<uint32_t>(a); }
}  // namespace hv
#define IFB_HV_DYNAMIC_SMEM(name_) unsigned char* const name_ = emu::smem

namespace ifbk {
#include "../../imageflow_b200/csrc/ifb_types.cuh"
#define HvTmap HvTmapDecl
#include "../../imageflow_b200/csrc/ifb_hv_kernel.cuh"
#undef HvTmap
}  // namespace ifbk

using namespace ifbk;
static_assert(sizeof(EmuTmap) == 128 && sizeof(HvTmapDecl) == 128, "descriptor size");
using KernelFn = void (*)(const JobDev*, const HvTmapDecl*, Tables, HvPlanDev, uint32_t, uint32_t*);
struct Pick { KernelFn fn; int threads; uint32_t (*smem)(uint32_t); };
template <int AV, int CH> static uint32_t smem_of(uint32_t low16) { return hv_total_bytes<AV, CH>(low16); }
static Pick pick(int av, int ch, int epi, int ori, int src) {      // epi: 0 general, 1 simple + linear, 2 simple + sRGB (as the engine picks them)
#define IFB_PICK_OS(AV_, CH_, O_, S_) if (av == AV_ && ch == CH_ && ori == O_ && src == S_) return Pick{epi == 1 ? hv_ring_kernel<AV_, CH_, 1, O_, S_> : \
        epi == 2 ? hv_ring_kernel<AV_, CH_, 2, O_, S_> : hv_ring_kernel<AV_, CH_, 0, O_, S_>, HvCfg<AV_, CH_>::kThreads, smem_of<AV_, CH_>};
#define IFB_PICK(AV_, CH_) IFB_PICK_OS(AV_, CH_, HV_ORI_FLIP, HV_SRC_RGBA) IFB_PICK_OS(AV_, CH_, HV_ORI_FLIP, HV_SRC_RGB24) \
                           IFB_PICK_OS(AV_, CH_, HV_ORI_TRANSPOSE, HV_SRC_RGBA) IFB_PICK_OS(AV_, CH_, HV_ORI_TRANSPOSE, HV_SRC_RGB24)
    IFB_PICK(4, 3) IFB_PICK(4, 4) IFB_PICK(6, 3) IFB_PICK(6, 4)
    return Pick{nullptr, 0, nullptr};
}

extern "C" uint32_t emu_hv_sizeof_jobdev(void) { return (uint32_t)sizeof(JobDev); }

// One launch of hv_ring_kernel<av, ch, simple, ori, src> (ori: HV_ORI_FLIP or HV_ORI_TRANSPOSE; src: HV_SRC_RGBA or HV_SRC_RGB24) with
// `grid` CTAs.  `blob` = the tables of ifb200_hv_plan_tables for the ORIENTED geometry (offsets in o[7]: strips, hw, hdone, vw, vdone,
// bands, total; dims4 = the oriented in_w, in_h, out_w, out_h and the weight records per strip = info.cap_px); in_ptrs[i] /
// in_whs[i*3..] describe job i's tensor of the STORED rows (16-byte aligned base, elements per row, rows, stride in bytes); the jobs'
// flags carry JF_FLIP_X / JF_FLIP_Y.  sb_low16: where dynamic shared memory starts in the emulated shared window.  Returns the number
// of bad accesses (0 = clean), or -1 for a form that does not exist.
extern "C" int emu_hv_launch_rows_oriented(int av, int ch, int simple, int ori, int src, unsigned grid, const void* jobs, uint32_t n_jobs,
                                           const uint8_t* const* in_ptrs, const uint32_t* in_whs, const float* t_lin, const float* t_srgb,
                                           const uint8_t* lut16k, const uint8_t* blob, const uint64_t* o, const uint32_t* dims4, int n_strips,
                                           int n_bands, uint32_t sb_low16) {
    const Pick pk = pick(av, ch, simple ? ((static_cast<const JobDev*>(jobs)[0].flags & JF_LINEAR) ? 1 : 2) : 0, ori, src);
    if (!pk.fn) return -1;
    std::vector<EmuTmap> tms(n_jobs);
    for (uint32_t i = 0; i < n_jobs; ++i) {
        tms[i] = EmuTmap{}; tms[i].base = in_ptrs[i]; tms[i].w = in_whs[i * 3]; tms[i].h = in_whs[i * 3 + 1]; tms[i].stride = in_whs[i * 3 + 2];
        tms[i].bytes = src == HV_SRC_RGB24; tms[i].transposed = ori == HV_ORI_TRANSPOSE;
        if ((uintptr_t)in_ptrs[i] & 15) return -1;
    }
    HvPlanDev pl{};
    pl.in_w = dims4[0]; pl.in_h = dims4[1]; pl.out_w = dims4[2]; pl.out_h = dims4[3]; pl.hw_stride = dims4[4];
    pl.n_strips = n_strips; pl.n_bands = n_bands;
    pl.strips = reinterpret_cast<const HvStripDev*>(blob + o[0]);
    pl.hw = reinterpret_cast<const float*>(blob + o[1]); pl.hdone = blob + o[2];
    pl.vw = reinterpret_cast<const float*>(blob + o[3]); pl.vdone = blob + o[4];
    pl.bands = reinterpret_cast<const HvBandDev*>(blob + o[5]);
    const Tables tb{t_lin, t_srgb, lut16k};
    std::vector<uint32_t> counters((size_t)n_strips, 0u);
    const size_t smem_bytes = pk.smem(sb_low16);
    const int nthreads = pk.threads, nwarps = nthreads / 32;
    emu::gridDim = {grid, 1, 1};
    emu::bad_access = 0;
    for (unsigned b = 0; b < grid; ++b) {
        emu::blockIdx = {b, 0, 0};
        std::unique_ptr<unsigned char, decltype(&std::free)> sm(static_cast<unsigned char*>(std::aligned_alloc(1024, (smem_bytes + 1023) / 1024 * 1024)), &std::free);
        std::memset(sm.get(), 0xFF, smem_bytes);
        emu::smem = sm.get(); emu::smem_bytes = smem_bytes; emu::win_base = 0x01000000u + sb_low16;
        std::barrier<> bb(nthreads);
        emu::block_barrier = &bb;
        std::vector<std::unique_ptr<std::barrier<>>> wb;
        for (int w = 0; w < nwarps; ++w) { wb.emplace_back(new std::barrier<>(32)); emu::warp_barrier[w] = wb.back().get(); }
        std::vector<std::thread> th;
        for (unsigned t = 0; t < (unsigned)nthreads; ++t)
            th.emplace_back([=, &tms, &counters] {
                emu::threadIdx = {t, 0, 0};
                pk.fn(static_cast<const JobDev*>(jobs), reinterpret_cast<const HvTmapDecl*>(tms.data()), tb, pl, n_jobs, counters.data());
            });
        for (auto& x : th) x.join();
    }
    return emu::bad_access.load();
}
