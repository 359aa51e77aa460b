// cuda_emu.h -- what every CPU emulator of a product kernel needs to compile the kernel's CUDA source with g++: the keywords, the
// thread and block indices, the vector types with CUDA's alignment, and the intrinsics mapped onto IEEE host operations (the emulators
// are built with -ffp-contract=off, so nothing is fused that the kernel does not fuse with __fmaf_rn).
// TEST INFRASTRUCTURE: nothing in the product includes it.  Each *_kernel_emu.cc includes it first, then adds what is its own: how
// threads, barriers and shared memory run, and its IFB_<OP>_LOAD / STORE bindings.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __launch_bounds__(...)

namespace emu {
struct Idx { unsigned x, y, z; };
// Per OS thread: the threaded emulators run each CUDA thread of a CTA on an OS thread of its own, the sequential ones set it before
// each thread's call.  The others are set once per CTA or launch, before its threads run.
inline thread_local Idx threadIdx;
inline Idx blockIdx, blockDim, gridDim;
}  // namespace emu
using emu::blockDim;
using emu::blockIdx;
using emu::gridDim;
using emu::threadIdx;

// A 16-byte access of a kernel at an address that is not 16-byte aligned faults on the GPU; with these types it is undefined here too.
struct alignas(16) uint4 { uint32_t x, y, z, w; };
struct alignas(16) float4 { float x, y, z, w; };
struct alignas(8) float2 { float x, y; };
static inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return uint4{x, y, z, w}; }
static inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
static inline float2 make_float2(float x, float y) { return float2{x, y}; }

using std::max;
using std::min;
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline float __fmaf_rn(float a, float b, float c) { return std::fmaf(a, b, c); }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline float __fsub_rn(float a, float b) { return a - b; }
static inline float __fdiv_rn(float a, float b) { return a / b; }
static inline float __fsqrt_rn(float a) { return std::sqrt(a); }
static inline double __ddiv_rn(double a, double b) { return a / b; }
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline float __uint2float_rn(unsigned v) { return (float)v; }
static inline uint32_t __float_as_uint(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
static inline float __uint_as_float(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
static inline float2 __fadd2_rn(float2 a, float2 b) { return float2{a.x + b.x, a.y + b.y}; }
static inline float __fadd_rz(float a, float b) {          // add.rz.f32 without touching the thread's rounding mode (the compiler
    const double s = (double)a + (double)b;                  // may move arithmetic across fesetround): the double sum is exact
    float f = (float)s;                                      // for the operands met here; then round it toward zero
    if (std::fabs((double)f) > std::fabs(s)) f = std::nextafterf(f, 0.0f);
    return f;
}
static inline unsigned __float2uint_rz(float s) {           // cvt.rzi.u32.f32: NaN -> 0, saturating
    if (!(s > 0.0f)) return 0u;
    if (s >= 4294967296.0f) return 0xffffffffu;
    return (unsigned)s;
}
static inline uint32_t __byte_perm(uint32_t x, uint32_t y, uint32_t s) {
    const uint64_t v = ((uint64_t)y << 32) | x; uint32_t r = 0;
    for (int i = 0; i < 4; ++i) r |= (uint32_t)((v >> (8 * ((s >> (4 * i)) & 7))) & 0xff) << (8 * i);
    return r;
}
static inline int __ffs(int v) { return __builtin_ffs(v); }
