// Host emulation shim for running a CUDA kernel's SOURCE on the CPU (test infrastructure only).
//
// One CTA = one group of std::threads; __syncthreads() is a std::barrier over the CTA; threadIdx / blockIdx are
// thread-local; `extern __shared__` storage is a static buffer owned by the harness (CTAs run one after another).
// Only what the emulated kernels use is provided (no warp intrinsics, no inline PTX, no TMA / wgmma): it checks
// index arithmetic, barrier placement, shared-memory data flow and the numerical formulation -- not performance and
// not the PTX-level features.  Kernels opt in with `#ifdef B2D_HOST_EMU` around their CUDA-only includes and launcher.
#pragma once
#include <algorithm>
#include <barrier>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <functional>
#include <thread>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __shared__
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))

struct float2 { float x, y; };
struct alignas(16) float4 { float x, y, z, w; };
struct uint2 { uint32_t x, y; };
struct uint4 { uint32_t x, y, z, w; };
struct dim3 { unsigned x = 1, y = 1, z = 1; };
inline float2 make_float2(float x, float y) { return {x, y}; }
inline float4 make_float4(float x, float y, float z, float w) { return {x, y, z, w}; }
inline uint2 make_uint2(uint32_t x, uint32_t y) { return {x, y}; }
inline uint4 make_uint4(uint32_t x, uint32_t y, uint32_t z, uint32_t w) { return {x, y, z, w}; }

namespace emu {
inline thread_local dim3 t_idx, b_idx;
inline std::barrier<>* cta_barrier = nullptr;
inline void sync() { cta_barrier->arrive_and_wait(); }

// run `kernel` for every CTA of grid (gx, gy) with `threads` threads each, CTAs sequentially
inline void launch(unsigned gx, unsigned gy, unsigned threads, const std::function<void()>& kernel) {
    for (unsigned by = 0; by < gy; ++by)
        for (unsigned bx = 0; bx < gx; ++bx) {
            std::barrier<> bar((std::ptrdiff_t)threads);
            cta_barrier = &bar;
            std::vector<std::thread> pool;
            pool.reserve(threads);
            for (unsigned t = 0; t < threads; ++t)
                pool.emplace_back([=, &kernel] {
                    t_idx.x = t; b_idx.x = bx; b_idx.y = by; b_idx.z = 0;   // the emulated grid is 2-D
                    kernel();
                });
            for (auto& th : pool) th.join();
        }
}
}  // namespace emu

#define threadIdx (emu::t_idx)
#define blockIdx (emu::b_idx)
#define __syncthreads() emu::sync()

template <class T> inline T __ldg(const T* p) { return *p; }
using std::max;
using std::min;
inline float cospif(float x) { return (float)std::cos(M_PI * (double)x); }
inline float sinpif(float x) { return (float)std::sin(M_PI * (double)x); }
inline void sincospif(float x, float* s, float* c) { *s = sinpif(x); *c = cospif(x); }
inline uint32_t __umulhi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }

// IEEE single operations (build with -ffp-contract=off so the host compiler does not fuse them) and the fast-math
// intrinsics (libm accuracy instead of the SFU's: the emulated tests compare with tolerances that cover both)
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline float __fdividef(float a, float b) { return a / b; }
inline float __sinf(float x) { return std::sin(x); }
inline float __cosf(float x) { return std::cos(x); }
inline float __expf(float x) { return std::exp(x); }
inline float __logf(float x) { return std::log(x); }
inline void __sincosf(float x, float* s, float* c) { *s = std::sin(x); *c = std::cos(x); }

#define B2D_PI_F 3.14159265358979323846f
#define B2D_TWO_PI_F 6.28318530717958647692f

namespace b2d {
inline void st_global_v4(float* p, float4 v) { std::memcpy(p, &v, sizeof v); }
// same Philox4x32-10 construction as csrc/b2d_common.cuh (the emulated tests feed explicit noise; kept for linking)
inline uint4 philox4x32_10(uint4 c, uint2 k) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x, hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += W0; k.y += W1;
    }
    return c;
}
inline float4 philox_uniform_pm1(uint64_t seed, uint64_t utt, uint32_t quad) {
    const uint4 r = philox4x32_10(make_uint4(quad, 0u, (uint32_t)utt, (uint32_t)(utt >> 32)),
                                  make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const float s = 1.0f / 8388608.0f;
    return make_float4((float)(r.x >> 8) * s - 1.0f, (float)(r.y >> 8) * s - 1.0f, (float)(r.z >> 8) * s - 1.0f,
                       (float)(r.w >> 8) * s - 1.0f);
}
}  // namespace b2d
