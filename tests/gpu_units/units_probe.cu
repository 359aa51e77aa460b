// units_probe.cu -- TEST INFRASTRUCTURE: small kernels that call the product's own __device__ functions (ifb_kernels.cuh) on
// arrays, so that tests/test_store_units_gpu.py can hold every form of the store epilogue, as compiled for sm_90a with the
// product's flags (imageflow_b200/csrc/nvflags.mk), to exact references.
//
// Scalar checks count on the device: every check owns a Report (trials, mismatches, the first 16 counterexamples) and the
// references are computed in float64 next to the unit under test.  Float64 is exact for what is asked of it here:
//   * a float quotient or reciprocal rounded through double is the correctly rounded float one (53 >= 2 * 24 + 2);
//   * v * 16383 and v * 255 are exact in double, so (float) of them is RN32 of the product;
//   * (double)x + 0.5 is exact for every float x that can round to a byte other than 0 or 255.
#include "ifb_kernels.cuh"

using namespace ifbk;

struct Report {                                // 72 words; tests/gpu_units/__init__.py reads it back (outside the anonymous
    unsigned long long trials, bad;            // namespace: the extern "C" launchers that take it must stay exported)
    uint32_t n_ex, pad[3];
    uint32_t ex[16][4];                        // (operand a, operand b, got, expected) as raw bits
};
static_assert(sizeof(Report) == 72 * 4, "Report layout");

namespace {

__device__ __forceinline__ void note(Report* r, unsigned long long& bad, uint32_t a, uint32_t b, uint32_t got, uint32_t want) {
    ++bad;
    if (*reinterpret_cast<volatile uint32_t*>(&r->n_ex) < 16u) {
        const uint32_t k = atomicAdd(&r->n_ex, 1u);
        if (k < 16u) { r->ex[k][0] = a; r->ex[k][1] = b; r->ex[k][2] = got; r->ex[k][3] = want; }
    }
}
__device__ __forceinline__ void flush(Report* r, unsigned long long trials, unsigned long long bad) {
    if (trials) atomicAdd(&r->trials, trials);
    if (bad) atomicAdd(&r->bad, bad);
}

__device__ __forceinline__ uint64_t mix(uint64_t z) {             // splitmix64 finaliser: counter -> random bits
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ float fbits(uint32_t u) { return __uint_as_float(u); }
__device__ __forceinline__ uint32_t ubits(float f) { return __float_as_uint(f); }
__device__ __forceinline__ bool same(float a, float b) { return ubits(a) == ubits(b); }
// a float with the given sign bit, unbiased exponent (normal range) and random significand
__device__ __forceinline__ float make_float(uint32_t sign, int e, uint32_t sig) { return fbits((sign << 31) | ((uint32_t)(e + 127) << 23) | (sig & 0x7fffffu)); }

// ---------------------------------------------------------------- exact references
__device__ __forceinline__ float div_ref(float x, float d) { return (float)((double)x / (double)d); }
// color.rs:101-108 by its definition: trunc(x + 0.5) saturated to [0, 255], NaN -> 0
__device__ __forceinline__ uint32_t clamp_ref(float x) {
    if (x != x) return 0u;
    const double t = trunc((double)x + 0.5);
    return t <= 0.0 ? 0u : t >= 255.0 ? 255u : (uint32_t)t;
}
// lut.rs:4-8: the table index clamp(RN32(v * 16383), 0, 16383) truncated, NaN -> 0
__device__ __forceinline__ uint32_t index_ref(float v) {
    if (v != v) return 0u;
    const double s = (double)(float)((double)v * 16383.0);
    return s <= 0.0 ? 0u : s >= 16383.0 ? 16383u : (uint32_t)trunc(s);
}
__device__ __forceinline__ uint32_t srgb_ref(float v) { return clamp_ref((float)((double)v * 255.0)); }

#define kInf __int_as_float(0x7f800000)
constexpr uint32_t kGuardLo = 0x30000000u, kGuardN = 0x20000000u;     // t2_div3's guard: 2^-31 <= d < 2^33
__device__ __forceinline__ bool markstein_exception(uint32_t db) { return (db & 0x7fffffu) == 0x7fffffu; }
// numerators for which t2_div3 claims the correctly rounded quotient: 2^-100 <= |x| < 2^64 (and 0)
__device__ __forceinline__ bool numerator_in_range(float x) { const uint32_t a = ubits(x) & 0x7fffffffu; return a == 0u || (a >= 0x0d800000u && a < 0x5f800000u); }

// ---------------------------------------------------------------- reciprocal: every d of the guard
__global__ void rcp_kernel(Report* in_guard, Report* excluded) {
    unsigned long long t0 = 0, b0 = 0, t1 = 0, b1 = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < kGuardN; i += gridDim.x * blockDim.x) {
        const uint32_t db = kGuardLo + i;
        const float d = fbits(db);
        const float got = t2_rcp_inrange(d), want = div_ref(1.0f, d);
        if (markstein_exception(db)) { ++t1; if (!same(got, want)) note(excluded, b1, db, 0u, ubits(got), ubits(want)); }
        else { ++t0; if (!same(got, want)) note(in_guard, b0, db, 0u, ubits(got), ubits(want)); }
    }
    flush(in_guard, t0, b0); flush(excluded, t1, b1);
}

// ---------------------------------------------------------------- quotient t2_div3 over the guarded divisors
// MODE 0: numerators next to a rounding midpoint of a random quotient q: x = RN((q + ulp(q)/2) * d) and its two neighbours.
// MODE 1: three random numerators, |x| in [2^-100, 2^64), both signs.
// MODE 2: three numerators below 2^-100 in magnitude (subnormals and zeros included): the encoded bytes of both encodings
//         must equal those of the IEEE quotient (ifb_tile2_kernel.cuh: the residual may be inexact there).
template <int MODE>
__global__ void div3_kernel(Report* r, uint64_t seed, const uint8_t* __restrict__ idx_lo, const uint8_t* __restrict__ idx_hi) {
    unsigned long long trials = 0, bad = 0;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < kGuardN; i += gridDim.x * blockDim.x) {
        const uint32_t db = kGuardLo + i;
        if (markstein_exception(db)) continue;
        const float d = fbits(db);
        const uint64_t h0 = mix(seed ^ ((uint64_t)i << 2)), h1 = mix(seed ^ ((uint64_t)i << 2 | 1u));
        float x[3];
        if (MODE == 0) {
            const float q = make_float((uint32_t)(h0 >> 63), -68 + (int)((h0 >> 32) % 99u), (uint32_t)h0);
            const double ulp = (double)(nextafterf(fabsf(q), kInf) - fabsf(q));
            const double m = (double)q + copysign(0.5 * ulp, (double)q);          // exact: 25 significant bits
            x[0] = (float)(m * (double)d);                                        // m * d is exact in double
            x[1] = nextafterf(x[0], -kInf); x[2] = nextafterf(x[0], kInf);
        } else if (MODE == 1) {
            for (int k = 0; k < 3; ++k) {
                const uint64_t h = k == 0 ? h0 : k == 1 ? h1 : mix(h0 ^ h1);
                x[k] = make_float((uint32_t)(h >> 63), -100 + (int)((h >> 32) % 164u), (uint32_t)h);
            }
        } else {
            for (int k = 0; k < 3; ++k) {
                const uint64_t h = k == 0 ? h0 : k == 1 ? h1 : mix(h0 ^ h1);
                const uint32_t mag = (uint32_t)(h % 0x0d800000ull);              // every pattern below 2^-100, 0 and subnormals included
                x[k] = fbits(((uint32_t)(h >> 63) << 31) | mag);
            }
        }
        float2 x01 = make_float2(x[0], x[1]);
        float x2 = x[2];
        t2_div3(x01, x2, d);
        const float got[3] = {x01.x, x01.y, x2};
        for (int k = 0; k < 3; ++k) {
            if (MODE != 2 && !numerator_in_range(x[k])) continue;
            ++trials;
            if (MODE != 2) {
                const float want = div_ref(x[k], d);
                if (!same(got[k], want)) note(r, bad, ubits(x[k]), db, ubits(got[k]), ubits(want));
            } else {
                const float ieee = __fdiv_rn(x[k], d);
                const uint32_t g = encode_sm<false>(nullptr, got[k]) | encode_sm<true>(idx_lo, got[k]) << 8 | encode_sm<true>(idx_hi, got[k]) << 16;
                const uint32_t w = encode_sm<false>(nullptr, ieee) | encode_sm<true>(idx_lo, ieee) << 8 | encode_sm<true>(idx_hi, ieee) << 16;
                if (g != w) note(r, bad, ubits(x[k]), db, g, w);
            }
        }
    }
    flush(r, trials, bad);
}

// every (x, d) pair of two lists against __fdiv_rn (NaN: only NaN-ness is compared).  For a divisor inside the guard the lists
// hold numerators of t2_div3's domain only (+0 or 2^-100 <= |x| < 2^64; below that see div3_kernel<2>)
__global__ void div3_edges_kernel(Report* r, const float* __restrict__ ds, uint32_t nd, const float* __restrict__ xs, uint32_t nx) {
    unsigned long long trials = 0, bad = 0;
    const uint64_t n = (uint64_t)nd * nx;
    for (uint64_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const float d = ds[i / nx], x = xs[i % nx];
        float2 x01 = make_float2(x, x);
        float x2 = x;
        t2_div3(x01, x2, d);
        const float got[3] = {x01.x, x01.y, x2};
        const float want = __fdiv_rn(x, d);
        for (int k = 0; k < 3; ++k) {                    // the same numerator in each of the three slots
            ++trials;
            const bool ok = (want != want) ? got[k] != got[k] : same(got[k], want);
            if (!ok) note(r, bad, ubits(x), ubits(d), ubits(got[k]), ubits(want));
        }
    }
    flush(r, trials, bad);
}

// ---------------------------------------------------------------- clamps: all 2^32 float patterns
__global__ void clamp_kernel(Report* r_ff, Report* r_rz) {
    unsigned long long trials = 0, b0 = 0, b1 = 0;
    for (uint64_t i = blockIdx.x * blockDim.x + threadIdx.x; i < (1ull << 32); i += (uint64_t)gridDim.x * blockDim.x) {
        const float x = fbits((uint32_t)i);
        const uint32_t want = clamp_ref(x), g0 = uchar_clamp_ff(x), g1 = uchar_clamp_ff_rz(x);
        ++trials;
        if (g0 != want) note(r_ff, b0, (uint32_t)i, 0u, g0, want);
        if (g1 != want) note(r_rz, b1, (uint32_t)i, 0u, g1, want);
    }
    flush(r_ff, trials, b0); flush(r_rz, trials, b1);
}

// ---------------------------------------------------------------- encoders: all 2^32 float patterns
// The linear encoders are run on tables that hold their own index (idx_lo[i] = i & 255, idx_hi[i] = i >> 8), so that the
// table INDEX is compared, not the byte.  Reports: 0 lut_encode, 1 ring kernel (hv_finish_pixel<1, 3>), 2 encode_sm<true>,
// 3 encode(false) (generic pair), 4 ring kernel sRGB (hv_finish_pixel<2, 3>), 5 encode_sm<false>.
constexpr int kEncThreads = 256;
__global__ void __launch_bounds__(kEncThreads) encode_kernel(Report* r, const uint8_t* __restrict__ idx_lo, const uint8_t* __restrict__ idx_hi,
                                                             const float* __restrict__ t_any) {
    extern __shared__ __align__(16) unsigned char sm[];
    // two LUT blocks of the ring kernel (64 KB each: index tables as its linear->sRGB table), then the tile kernel's two tables
    const uint32_t blk_lo = hv::smem_u32(sm), blk_hi = blk_lo + 65536u;
    uint8_t* const s_lo = sm + 131072;
    uint8_t* const s_hi = s_lo + 16384;
    const int t = threadIdx.x;
    hv_fill_luts<kEncThreads>(blk_lo, Tables{t_any, t_any, idx_lo}, JF_LINEAR, t);
    hv_fill_luts<kEncThreads>(blk_hi, Tables{t_any, t_any, idx_hi}, JF_LINEAR, t);
    for (int i = t; i < 16384; i += kEncThreads) { s_lo[i] = idx_lo[i]; s_hi[i] = idx_hi[i]; }
    __syncthreads();
    const uint32_t lane4 = (uint32_t)(t & 31) * 4u;
    const JobDev job{};
    // the ring kernel encodes b, g, r alike and stores alpha 255: anything else counts as a mismatch (no reference is all ones)
    auto agree = [](uint32_t w) { return (w & 0xffu) == ((w >> 8) & 0xffu) && (w & 0xffu) == ((w >> 16) & 0xffu) && (w >> 24) == 255u; };
    unsigned long long trials = 0, bad[6] = {0, 0, 0, 0, 0, 0};
    for (uint64_t i = blockIdx.x * blockDim.x + t; i < (1ull << 32); i += (uint64_t)gridDim.x * blockDim.x) {
        const float v = fbits((uint32_t)i);
        const uint32_t wi = index_ref(v), ws = srgb_ref(v);
        ++trials;
        uint32_t g[6];
        g[0] = lut_encode(idx_lo, v) | lut_encode(idx_hi, v) << 8;
        const uint32_t hl = hv_finish_pixel<1, 3>(v, v, v, 0.0f, JF_LINEAR, job, blk_lo, blk_lo + lane4, nullptr);
        const uint32_t hh = hv_finish_pixel<1, 3>(v, v, v, 0.0f, JF_LINEAR, job, blk_hi, blk_hi + lane4, nullptr);
        g[1] = agree(hl) && agree(hh) ? (hl & 0xffu) | (hh & 0xffu) << 8 : 0xffffffffu;
        g[2] = encode_sm<true>(s_lo, v) | encode_sm<true>(s_hi, v) << 8;
        g[3] = encode(false, nullptr, v);
        const uint32_t hs = hv_finish_pixel<2, 3>(v, v, v, 0.0f, 0u, job, blk_lo, blk_lo + lane4, nullptr);
        g[4] = agree(hs) ? hs & 0xffu : 0xffffffffu;
        g[5] = encode_sm<false>(nullptr, v);
        for (int k = 0; k < 6; ++k) {
            const uint32_t want = k < 3 ? wi : ws;
            if (g[k] != want) note(r + k, bad[k], (uint32_t)i, 0u, g[k], want);
        }
    }
    for (int k = 0; k < 6; ++k) flush(r + k, trials, bad[k]);
}

// ---------------------------------------------------------------- store epilogues on arrays of (F, canvas pixel)
__device__ JobDev g_job;                       // the job every epilogue reads (matte, colour matrix), in global memory like the engine's

// finish_pixel<SIMPLE> (generic pair, ifb_finish.cuh): the canvas pixel is read where it lies
template <bool SIMPLE>
__global__ void fp_kernel(const float4* __restrict__ f, uint32_t* px, uint32_t n, Tables tb) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 v = f[i];
    px[i] = finish_pixel<SIMPLE>(v.x, v.y, v.z, v.w, g_job, tb, reinterpret_cast<const uint8_t*>(px + i));
}

// hv_finish_pixel<EPI, CH> with the LUT block as the ring kernel fills it
constexpr int kHvThreads = 256;
template <int EPI, int CH>
__global__ void __launch_bounds__(kHvThreads) hv_kernel(const float4* __restrict__ f, uint32_t* px, uint32_t n, Tables tb) {
    extern __shared__ __align__(16) unsigned char sm[];
    const uint32_t lut = hv::smem_u32(sm);
    hv_fill_luts<kHvThreads>(lut, tb, g_job.flags, threadIdx.x);
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float4 v = f[i];
    const uint32_t o = hv_finish_pixel<EPI, CH>(v.x, v.y, v.z, CH == 4 ? v.w : 0.0f, g_job.flags, g_job, lut, lut + (threadIdx.x & 31u) * 4u,
                                                reinterpret_cast<const uint8_t*>(px + i));
    px[i] = o;
}

// finish_pixel_sm<CH, LINEAR, COMPOSE, CM> with its tables in shared memory as fused_tile2_kernel stages them
template <int CH, bool LINEAR, int COMPOSE, bool CM>
__global__ void __launch_bounds__(256) sm_kernel(const float4* __restrict__ f, uint32_t* px, uint32_t n, Tables tb) {
    __shared__ float sT[256];
    __shared__ float sCm[20];
    __shared__ __align__(16) uint8_t sLut[16384];
    const int t = threadIdx.x;
    sT[t] = (LINEAR ? tb.t_lin : tb.t_srgb)[t];
    if (t < 20) sCm[t] = g_job.cm[t];
    for (int k = t; k < 16384; k += 256) sLut[k] = tb.lut16k[k];
    __syncthreads();
    const uint32_t i = blockIdx.x * blockDim.x + t;
    if (i >= n) return;
    float cm9[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (CM)
        for (int c = 0; c < 3; ++c) { cm9[c * 3] = sCm[c * 5]; cm9[c * 3 + 1] = sCm[c * 5 + 1]; cm9[c * 3 + 2] = sCm[c * 5 + 2]; }
    const float matte[4] = {g_job.matte[0], g_job.matte[1], g_job.matte[2], g_job.matte[3]};
    const float4 v = f[i];
    const uint32_t d = (COMPOSE == 1 && CH == 4) ? px[i] : 0u;
    px[i] = finish_pixel_sm<CH, LINEAR, COMPOSE, CM>(make_float2(v.x, v.y), v.z, CH == 4 ? v.w : 0.0f, g_job.flags, matte, sT, sLut, sCm, cm9, d);
}

using EpiFn = void (*)(const float4*, uint32_t*, uint32_t, Tables);
#define IFBU_SM_CM(CH_, LIN_, CO_) sm_kernel<CH_, LIN_, CO_, false>, sm_kernel<CH_, LIN_, CO_, true>
#define IFBU_SM_CO4(LIN_) IFBU_SM_CM(4, LIN_, 0), IFBU_SM_CM(4, LIN_, 1), IFBU_SM_CM(4, LIN_, 2)
#define IFBU_SM_CO3(LIN_) IFBU_SM_CM(3, LIN_, 0), IFBU_SM_CM(3, LIN_, 0), IFBU_SM_CM(3, LIN_, 0)
// the instantiations the engine compiles (ifb_engine.cu kTile2): without meaningful alpha every compositing mode is compose 0
const EpiFn kSm[2][2][6] = {{{IFBU_SM_CO3(false)}, {IFBU_SM_CO3(true)}}, {{IFBU_SM_CO4(false)}, {IFBU_SM_CO4(true)}}};   // [ch==4][linear][compose * 2 + cm]
const EpiFn kHv[3][2] = {{hv_kernel<0, 3>, hv_kernel<0, 4>}, {hv_kernel<1, 3>, hv_kernel<1, 4>}, {hv_kernel<2, 3>, hv_kernel<2, 4>}};

int blocks_for(const void* fn, int threads, size_t smem) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, threads, smem);
    return sms * (per_sm > 0 ? per_sm : 1);
}
int finish() { const cudaError_t e = cudaDeviceSynchronize(); return e == cudaSuccess ? (int)cudaGetLastError() : (int)e; }

}  // namespace

extern "C" {
// Every launcher runs on the legacy default stream, waits for the kernel and returns the cudaError_t.  Report* = device memory.
int ifbu_rcp(Report* in_guard, Report* excluded) {
    rcp_kernel<<<blocks_for((const void*)rcp_kernel, 256, 0), 256>>>(in_guard, excluded);
    return finish();
}
int ifbu_div3(int mode, Report* r, uint64_t seed, const uint8_t* idx_lo, const uint8_t* idx_hi) {
    if (mode == 0) div3_kernel<0><<<blocks_for((const void*)div3_kernel<0>, 256, 0), 256>>>(r, seed, idx_lo, idx_hi);
    else if (mode == 1) div3_kernel<1><<<blocks_for((const void*)div3_kernel<1>, 256, 0), 256>>>(r, seed, idx_lo, idx_hi);
    else if (mode == 2) div3_kernel<2><<<blocks_for((const void*)div3_kernel<2>, 256, 0), 256>>>(r, seed, idx_lo, idx_hi);
    else return (int)cudaErrorInvalidValue;
    return finish();
}
int ifbu_div3_edges(Report* r, const float* ds, uint32_t nd, const float* xs, uint32_t nx) {
    div3_edges_kernel<<<blocks_for((const void*)div3_edges_kernel, 256, 0), 256>>>(r, ds, nd, xs, nx);
    return finish();
}
int ifbu_clamp(Report* r_ff, Report* r_rz) {
    clamp_kernel<<<blocks_for((const void*)clamp_kernel, 256, 0), 256>>>(r_ff, r_rz);
    return finish();
}
int ifbu_encode(Report* r6, const uint8_t* idx_lo, const uint8_t* idx_hi, const float* t_any) {
    const size_t smem = 131072 + 2 * 16384;
    cudaError_t e = cudaFuncSetAttribute(encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    encode_kernel<<<blocks_for((const void*)encode_kernel, kEncThreads, smem), kEncThreads, smem>>>(r6, idx_lo, idx_hi, t_any);
    return finish();
}
// family 0: finish_pixel<a != 0> (b, c, d unused); family 1: hv_finish_pixel<EPI = a, CH = b>; family 2: finish_pixel_sm<CH = b,
// LINEAR = c, COMPOSE = a, CM = d>.  f: n float4 (b, g, r, a); px: n canvas pixels in, n results out.  job: flags, matte[4], cm[20].
int ifbu_epilogue(int family, int a, int b, int c, int d, const float4* f, uint32_t* px, uint32_t n, uint32_t flags, const float* matte,
                  const float* cm, const float* t_lin, const float* t_srgb, const uint8_t* lut16k) {
    JobDev job{};
    job.flags = flags;
    for (int k = 0; k < 4; ++k) job.matte[k] = matte[k];
    for (int k = 0; k < 20; ++k) job.cm[k] = cm[k];
    cudaError_t e = cudaMemcpyToSymbol(g_job, &job, sizeof job);
    if (e != cudaSuccess) return (int)e;
    const Tables tb{t_lin, t_srgb, lut16k};
    const unsigned grid = (n + 255u) / 256u;
    if (n == 0) return 0;
    if (family == 0) {
        if (a) fp_kernel<true><<<grid, 256>>>(f, px, n, tb);
        else fp_kernel<false><<<grid, 256>>>(f, px, n, tb);
    } else if (family == 1) {
        if (a < 0 || a > 2 || (b != 3 && b != 4)) return (int)cudaErrorInvalidValue;
        const EpiFn fn = kHv[a][b == 4];
        e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, 65536);
        if (e != cudaSuccess) return (int)e;
        fn<<<grid, kHvThreads, 65536>>>(f, px, n, tb);
    } else if (family == 2) {
        if (a < 0 || a > 2 || (b != 3 && b != 4) || (b == 3 && a != 0)) return (int)cudaErrorInvalidValue;
        kSm[b == 4][c != 0][a * 2 + (d != 0)]<<<grid, 256>>>(f, px, n, tb);
    } else {
        return (int)cudaErrorInvalidValue;
    }
    return finish();
}
}
