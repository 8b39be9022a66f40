// Host emulation shim for running a CUDA kernel's SOURCE on the CPU (test infrastructure only).
//
// One CTA = one group of std::threads; __syncthreads() is a std::barrier over the CTA; threadIdx / blockIdx are
// thread-local; `extern __shared__` storage is a static buffer owned by the driver (CTAs run one after another, except
// the CTAs of one thread-block cluster, which run together).  It checks index arithmetic, barrier placement,
// shared-memory data flow and the numerical formulation -- not performance.  Kernels opt in with `#ifdef B2D_HOST_EMU`
// around their CUDA-only includes, intrinsics and launchers.
//
// Besides the CTA it models (each written from the PTX ISA, not from the kernels that use it):
//   warps        32 consecutive threads of the CTA, each warp with its own barrier: __syncwarp, __shfl_xor_sync and
//                mma_tf32 are collectives of the 32 lanes (every lane must reach them, as the hardware requires).
//   mma_tf32     mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32: the lanes exchange their A, B and C fragments
//                and each computes its own D elements.  Operands are truncated to TF32 (low 13 mantissa bits cleared);
//                the 8 products and C are summed in double and rounded once to fp32.  The hardware accumulates with
//                truncation instead, so the emulator is more accurate in the last ulp: its tests bound indexing and
//                fragment layout, not the tensor cores' rounding.
//   cp.async     cp_async16 queues the copy in the issuing thread and poisons its destination (NaN bytes: the contents
//                are undefined until the wait); cp_async_commit closes a group; cp_async_wait<N> performs the copies
//                of every group but the N most recent, zero-filling the bytes at or past src_bytes.  A stage read
//                before its wait reads the poison, and a stage refilled while another thread still reads it is a
//                write TSan sees.  b2d::smem_u32 is an offset into the shared window the driver registered.
//   static __shared__  B2D_SHARED(T, name, dims) -- in the kernels `__shared__ T name dims` -- is one copy per
//                emulated CTA, in an arena allocated before its threads start and filled with NaN bytes.
//   clusters     launch(..., cluster) runs the CTAs of one cluster at the same time; cg::this_cluster() gives
//                block_rank(), sync() (one barrier over the cluster's threads) and map_shared_rank(p, q) (the same
//                offset in CTA q's copy of a B2D_SHARED array).
#pragma once
#include <algorithm>
#include <atomic>
#include <barrier>
#include <cassert>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <functional>
#include <memory>
#include <thread>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __restrict__
#define __shared__
#define __launch_bounds__(...)
#define __cluster_dims__(...)
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
inline thread_local dim3 t_idx, b_idx, grid_dim, block_dim;

struct Lane {                      // what one thread offers to its warp's collectives
    float f;
    int i;
    uint32_t a[4], b[2];
};
// Every lane runs the same sequence of collectives, so they alternate between two slot sets: a lane can be at most one
// collective ahead of another (each one ends in a warp barrier), and one barrier per collective suffices.
inline thread_local unsigned t_coll = 0;
// static __shared__ arrays (B2D_SHARED) of one CTA: each array site takes a fixed offset for the whole process
constexpr size_t kStaticArena = 48 * 1024;
inline std::atomic<size_t> static_top{0};
inline size_t reserve_static(size_t bytes) {
    const size_t off = static_top.fetch_add((bytes + 15) & ~(size_t)15, std::memory_order_relaxed);
    if (off + bytes > kStaticArena) {
        std::fprintf(stderr, "B2D_SHARED: more than %zu bytes of static shared arrays\n", kStaticArena);
        std::abort();
    }
    return off;
}

struct Cta {
    std::unique_ptr<std::barrier<>> bar;
    std::vector<std::unique_ptr<std::barrier<>>> warp_bar;
    std::vector<Lane> lanes;
    std::unique_ptr<unsigned char[]> arena;        // kStaticArena bytes, NaN-filled when the CTA starts
    unsigned rank = 0;
    void start(unsigned threads, unsigned r) {
        bar.reset(new std::barrier<>((std::ptrdiff_t)threads));
        warp_bar.clear();
        for (unsigned w = 0; w < threads; w += 32)                 // a last partial warp meets on its own
            warp_bar.emplace_back(new std::barrier<>((std::ptrdiff_t)std::min(32u, threads - w)));
        lanes.assign(2 * threads, Lane{});
        if (!arena) arena.reset(new unsigned char[kStaticArena]);
        std::memset(arena.get(), 0xFF, kStaticArena);
        rank = r;
    }
};
struct Cluster {
    std::barrier<>* bar = nullptr;
    std::vector<Cta>* ctas = nullptr;
};
inline thread_local Cta* t_cta = nullptr;
inline thread_local Cluster* t_cluster = nullptr;

inline void sync() { t_cta->bar->arrive_and_wait(); }
inline void warp_sync() { t_cta->warp_bar[t_idx.x >> 5]->arrive_and_wait(); }

// ---- cp.async: per-thread queue of committed groups ----
struct CpAsync { unsigned char* dst; const void* src; uint32_t bytes; };
inline thread_local std::vector<CpAsync> cp_open;
inline thread_local std::deque<std::vector<CpAsync>> cp_groups;
inline unsigned char* smem_window = nullptr;      // the shared buffer b2d::smem_u32 addresses
inline size_t smem_window_bytes = 0;
inline void shared_window(void* base, size_t bytes) { smem_window = (unsigned char*)base; smem_window_bytes = bytes; }

// run `kernel` for every CTA of `grid` with `threads` threads each; the CTAs of one cluster (`cluster` consecutive
// x indices) together, clusters one after another.  One std::thread per CUDA thread of a cluster serves every cluster of
// the launch in turn; all of them meet between two clusters, so each cluster starts after the previous one finished.
inline void launch(dim3 grid, unsigned threads, const std::function<void()>& kernel, unsigned cluster = 1) {
    assert(grid.x % cluster == 0);
    const unsigned per_x = grid.x / cluster, groups = per_x * grid.y * grid.z, n = threads * cluster;
    std::vector<Cta> ctas(cluster);
    std::barrier<> cbar((std::ptrdiff_t)n), between((std::ptrdiff_t)n);
    Cluster cl{&cbar, &ctas};
    for (unsigned q = 0; q < cluster; ++q) ctas[q].start(threads, q);
    std::vector<std::thread> pool;
    pool.reserve(n);
    for (unsigned q = 0; q < cluster; ++q)
        for (unsigned t = 0; t < threads; ++t)
            pool.emplace_back([=, &kernel, &ctas, &cl, &between] {
                t_idx = dim3{t, 0, 0};
                grid_dim = grid;
                block_dim = dim3{threads, 1, 1};
                t_cta = &ctas[q];
                t_cluster = &cl;
                for (unsigned g = 0; g < groups; ++g) {
                    if (g) {                                       // the previous cluster is done: fresh CTA state
                        between.arrive_and_wait();
                        if (t == 0) ctas[q].start(threads, q);
                        between.arrive_and_wait();
                    }
                    b_idx = dim3{(g % per_x) * cluster + q, (g / per_x) % grid.y, g / (per_x * grid.y)};
                    cp_open.clear();
                    cp_groups.clear();
                    t_coll = 0;
                    kernel();
                    cp_open.clear();
                    cp_groups.clear();
                }
            });
    for (auto& th : pool) th.join();
}
// the 2-D grid (gx, gy) of the older drivers
inline void launch(unsigned gx, unsigned gy, unsigned threads, const std::function<void()>& kernel) {
    launch(dim3{gx, gy, 1}, threads, kernel);
}

// one copy of a static __shared__ array per CTA, at the offset its site reserved on first use (no lock: the only
// synchronisation is the one-time initialisation of `off`)
template <class T, class Site>
T& cta_static(Site) {
    static const size_t off = reserve_static(sizeof(T));
    return *reinterpret_cast<T*>(t_cta->arena.get() + off);
}
}  // namespace emu

#define threadIdx (emu::t_idx)
#define blockIdx (emu::b_idx)
#define __syncthreads() emu::sync()
// `__shared__ T name dims` in device code (b2d_common.cuh)
#define B2D_SHARED(T, name, dims) T(&name) dims = emu::cta_static<T dims>([] {})

template <class T> inline T __ldg(const T* p) { return *p; }
using std::max;
using std::min;
inline float cospif(float x) { return (float)std::cos(M_PI * (double)x); }
inline float sinpif(float x) { return (float)std::sin(M_PI * (double)x); }
inline void sincospif(float x, float* s, float* c) { *s = sinpif(x); *c = cospif(x); }
inline uint32_t __umulhi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline uint32_t __float_as_uint(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }

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
inline float rsqrtf(float x) { return 1.0f / std::sqrt(x); }

// ---- warp collectives ----
inline void __syncwarp(unsigned = 0xffffffffu) { emu::warp_sync(); }
// the warp's slots of this collective (see t_coll)
inline emu::Lane* warp_slots() {
    return &emu::t_cta->lanes[(emu::t_coll++ & 1) * emu::block_dim.x + (threadIdx.x & ~31u)];
}
// every lane of the warp publishes its value, the warp meets, each reads lane ^ d's
inline float __shfl_xor_sync(unsigned, float v, int d) {
    emu::Lane* w = warp_slots();
    w[threadIdx.x & 31].f = v;
    emu::warp_sync();
    return w[(threadIdx.x & 31) ^ (unsigned)d].f;
}
inline int __shfl_xor_sync(unsigned, int v, int d) {
    emu::Lane* w = warp_slots();
    w[threadIdx.x & 31].i = v;
    emu::warp_sync();
    return w[(threadIdx.x & 31) ^ (unsigned)d].i;
}

// mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {d} = {a} x {b} + {d}.  Fragment layout (PTX ISA, "Matrix
// fragments for mma.m16n8k8", .tf32): with groupID = lane >> 2 and tig = lane % 4,
//   A (16 x 8, row):  a_i at row groupID + 8 (i % 2), column tig + 4 (i / 2)
//   B (8 x 8, col):   b_i at row (k) tig + 4 i, column (n) groupID
//   C, D (16 x 8):    c_i at row groupID + 8 (i / 2), column 2 tig + i % 2
inline void mma_tf32(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    const unsigned lane = threadIdx.x & 31;
    emu::Lane* w = warp_slots();
    std::memcpy(w[lane].a, a, sizeof a);
    w[lane].b[0] = b0;
    w[lane].b[1] = b1;
    emu::warp_sync();
    auto tf32 = [](uint32_t u) { return (double)__uint_as_float(u & 0xFFFFE000u); };
    auto A = [&](int r, int k) { return tf32(w[4 * (r % 8) + k % 4].a[(r / 8) + 2 * (k / 4)]); };
    auto Bm = [&](int k, int n) { return tf32(w[4 * n + k % 4].b[k / 4]); };
    const int gid = (int)lane >> 2, tig = (int)lane & 3;
    float out[4];
    for (int i = 0; i < 4; ++i) {
        const int r = gid + 8 * (i / 2), n = 2 * tig + i % 2;
        double s = (double)d[i];
        for (int k = 0; k < 8; ++k) s += A(r, k) * Bm(k, n);
        out[i] = (float)s;
    }
    for (int i = 0; i < 4; ++i) d[i] = out[i];
}

// ---- cp.async (mma_sync.cuh) ----
namespace b2d {
inline uint32_t smem_u32(const void* p) {
    const unsigned char* c = (const unsigned char*)p;
    if (!(c >= emu::smem_window && c < emu::smem_window + emu::smem_window_bytes)) {
        std::fprintf(stderr, "smem_u32: pointer outside the registered shared window\n");
        std::abort();
    }
    return (uint32_t)(c - emu::smem_window);
}
}  // namespace b2d
inline void cp_async16(uint32_t dst, const void* src, uint32_t src_bytes) {
    if ((dst & 15u) || dst + 16 > emu::smem_window_bytes || src_bytes > 16) {
        std::fprintf(stderr, "cp_async16: misaligned or out-of-window destination %u (%u bytes)\n", dst, src_bytes);
        std::abort();
    }
    unsigned char* p = emu::smem_window + dst;
    std::memset(p, 0xFF, 16);
    emu::cp_open.push_back({p, src, src_bytes});
}
inline void cp_async_commit() {
    emu::cp_groups.push_back(std::move(emu::cp_open));
    emu::cp_open.clear();
}
template <int N>
inline void cp_async_wait() {
    while (emu::cp_groups.size() > (size_t)N) {
        for (const auto& c : emu::cp_groups.front()) {
            std::memset(c.dst, 0, 16);
            if (c.bytes) std::memcpy(c.dst, c.src, c.bytes);
        }
        emu::cp_groups.pop_front();
    }
}

// ---- thread-block clusters (cooperative_groups) ----
namespace cooperative_groups {
struct cluster_group {
    unsigned block_rank() const { return emu::t_cta->rank; }
    void sync() const { emu::t_cluster->bar->arrive_and_wait(); }
    // p: an element of a B2D_SHARED array of this CTA -> the same offset in CTA q's arena (no lock)
    template <class T>
    T* map_shared_rank(T* p, unsigned q) const {
        const unsigned char *c = (const unsigned char*)p, *base = emu::t_cta->arena.get();
        if (c < base || c + sizeof(T) > base + emu::kStaticArena) {
            std::fprintf(stderr, "map_shared_rank: not a B2D_SHARED array\n");
            std::abort();
        }
        return reinterpret_cast<T*>((*emu::t_cluster->ctas)[q].arena.get() + (c - base));
    }
};
inline cluster_group this_cluster() { return {}; }
}  // namespace cooperative_groups

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
