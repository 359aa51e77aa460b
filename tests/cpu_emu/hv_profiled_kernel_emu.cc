// Runs the PROFILED forms of imageflow_b200/csrc/ifb_hv_kernel.cuh -- hv_ring_profiled_kernel<AV, CH, EPI, ORI, SRC, PROF>, the
// product's CUDA source unmodified -- on the CPU, with the primitives and the TMA emulation of hv_rows_oriented_kernel_emu.cc (one OS
// thread per CUDA thread, all four tensor maps with zero fill, box origins checked to be 16-byte aligned, mbarrier phases checked,
// shared memory as an exactly-sized heap block).  The plan (a ProfDev) follows the job array, as the engine uploads it.  Also the
// host side of ifb200_batch_enqueue_profiled's planning: ifb::ProfilePlans, and the plans transform_to_srgb_prepare gives through it.
// Built with -ffp-contract=off; with -fsanitize=address a run is also a memory check of the kernel.
// TEST INFRASTRUCTURE: nothing in the product calls this; the GPU remains the place where the kernel is run and timed.
#include "hv_rows_oriented_kernel_emu.cc"

#include "../../imageflow_b200/csrc/ifb_profile.h"

template <int AV, int CH, int PROF> static uint32_t smem_of_prof(uint32_t low16) { return hv_total_bytes<AV, CH, PROF>(low16); }
// The forms compiled here: matrix plans with both simple store epilogues, gray plans with the linear one, every ring depth, channel
// count, orientation class and source format.
static Pick pick_profiled(int av, int ch, int epi, int ori, int src, int prof) {
#define IFB_PICK_P(AV_, CH_, O_, S_) \
    if (av == AV_ && ch == CH_ && ori == O_ && src == S_) { \
        if (prof == PF_MATRIX && epi == 1) return Pick{hv_ring_profiled_kernel<AV_, CH_, 1, O_, S_, PF_MATRIX>, HvCfg<AV_, CH_, PF_MATRIX>::kThreads, smem_of_prof<AV_, CH_, PF_MATRIX>}; \
        if (prof == PF_MATRIX && epi == 2) return Pick{hv_ring_profiled_kernel<AV_, CH_, 2, O_, S_, PF_MATRIX>, HvCfg<AV_, CH_, PF_MATRIX>::kThreads, smem_of_prof<AV_, CH_, PF_MATRIX>}; \
        if (prof == PF_GRAY && epi == 1) return Pick{hv_ring_profiled_kernel<AV_, CH_, 1, O_, S_, PF_GRAY>, HvCfg<AV_, CH_, PF_GRAY>::kThreads, smem_of_prof<AV_, CH_, PF_GRAY>}; \
        return Pick{nullptr, 0, nullptr}; }
#define IFB_PICK_S(AV_, CH_, O_) IFB_PICK_P(AV_, CH_, O_, HV_SRC_BGRA) IFB_PICK_P(AV_, CH_, O_, HV_SRC_RGBA) IFB_PICK_P(AV_, CH_, O_, HV_SRC_RGB24)
#define IFB_PICK_O(AV_, CH_) IFB_PICK_S(AV_, CH_, HV_ORI_NONE) IFB_PICK_S(AV_, CH_, HV_ORI_FLIP) IFB_PICK_S(AV_, CH_, HV_ORI_TRANSPOSE)
    IFB_PICK_O(4, 3) IFB_PICK_O(4, 4) IFB_PICK_O(6, 3) IFB_PICK_O(6, 4)
    return Pick{nullptr, 0, nullptr};
}

extern "C" uint32_t emu_sizeof_profdev(void) { return (uint32_t)sizeof(ProfDev); }

// One launch of hv_ring_profiled_kernel<av, ch, epi, ori, src, prof> with `grid` CTAs; `jobs` = n_jobs JobDev followed by one ProfDev.
// Everything else as emu_hv_launch_rows_oriented (in_whs: elements per row, rows and stride of each job's STORED tensor; bytes for
// RGB24, pixels otherwise).  Returns the number of bad accesses (0 = clean), or -1 for a form that does not exist here.
extern "C" int emu_hv_launch_profiled(int av, int ch, int epi, int ori, int src, int prof, unsigned grid, const void* jobs, uint32_t n_jobs,
                                      const uint8_t* const* in_ptrs, const uint32_t* in_whs, const float* t_lin, const float* t_srgb,
                                      const uint8_t* lut16k, const uint8_t* blob, const uint64_t* o, const uint32_t* dims4, int n_strips,
                                      int n_bands, uint32_t sb_low16) {
    const Pick pk = pick_profiled(av, ch, epi, ori, src, prof);
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

// ifb::ProfilePlans over n profiles in order: plan_of[i] = the plan index of profile i, kinds[k] the kind of plan k.  Returns the number
// of plans, or -(i + 1) when profile i is refused (why gets the reason).
extern "C" int emu_profile_plans(const ifb200_source_profile* const* p, size_t n, uint32_t* plan_of, int32_t* kinds, char* why, size_t cap) {
    ifb::ProfilePlans pp;
    for (size_t i = 0; i < n; ++i) {
        std::string w;
        if (pp.add(*p[i], &plan_of[i], &w) != IFB200_OK) { std::snprintf(why, cap, "%s", w.c_str()); return -(int)(i + 1); }
    }
    for (size_t k = 0; k < pp.plans.size(); ++k) kinds[k] = pp.plans[k].kind;
    return (int)pp.plans.size();
}

// transform_to_srgb_prepare over n 1x1 BGRA jobs (not in place) with these profiles: plan_of[i] = the plan index of job i's item.
// Returns the number of plans, or -1 with why.
extern "C" int emu_transform_plan_of(const ifb200_source_profile* const* p, size_t n, uint32_t* plan_of, char* why, size_t cap) {
    static uint8_t src[4], dst[4];
    std::vector<ifb200_to_srgb_desc> d(n);
    for (size_t i = 0; i < n; ++i) d[i] = ifb200_to_srgb_desc{IFB200_PROFILE_SRC_BGRA, src, 4, dst, 4, 1, 1, p[i]};
    ifb::PfWork wk;
    int code = 0;
    const std::string w = ifb::transform_to_srgb_prepare(d.data(), n, wk, &code);
    if (!w.empty()) { std::snprintf(why, cap, "%s", w.c_str()); return -1; }
    for (size_t i = 0; i < wk.plan_of.size(); ++i) plan_of[i] = wk.plan_of[i] & ~ifb::kPfBgra;
    return (int)wk.plans.size();
}
