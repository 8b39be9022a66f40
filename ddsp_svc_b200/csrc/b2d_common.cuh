// Shared host/device helpers for libb200ddsp (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>

#include "../../include/b200ddsp.h"

// ---------------------------------------------------------------------------------------
// host side: thread-local error string, launch check
// ---------------------------------------------------------------------------------------
namespace b2d {

// SM count of the current device (cached per device; 132 on the H100 SXM): the launch heuristics size grids and chunk
// lengths so that a launch fills one or a few waves
int num_sms();

char* err_buf();                                   // thread-local, defined in api.cu
int   fail(int code, const char* fmt, ...);       // formats into err_buf, returns code

inline int check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return fail((int)e, "%s: %s", what, cudaGetErrorString(e));
    return 0;
}

// b2d_set_fft_arith(1): the FFT kernels (ltv_fir_fft, superfast, combsubfast) use their "packed" instantiations
extern std::atomic<int> g_fft_packed;   // debug A/B switch (b2d_set_fft_arith), read once per call
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

inline size_t align256(size_t bytes) { return (bytes + 255) / 256 * 256; }
inline float* ws_at(void* ws, size_t off) { return reinterpret_cast<float*>(static_cast<char*>(ws) + off); }
inline const float* ws_at(const void* ws, size_t off) {
    return reinterpret_cast<const float*>(static_cast<const char*>(ws) + off);
}
// appends a buffer of `floats` floats to a workspace of `bytes` bytes (each buffer 256-byte aligned) -> its offset
inline size_t ws_append(size_t& bytes, size_t floats) {
    const size_t off = bytes;
    bytes += align256(floats * 4);
    return off;
}

// Forward workspaces of b2d_sins_synth / b2d_combsub_synth.  The backwards read the forward's buffers back from them, so
// the drivers, the workspace queries and the backwards all take their byte offsets from here.  bytes == 0: bad shape.
size_t fir_spec_floats(int B, int nF);     // ltv_fir_fft.cu: one filter's packed spectra
// sinusoids [B, T] | ir_allpass [B, nF, 2 (Ma - 1)] | ir_noise [B, nF, 2 (Mn - 1)]; with `spectrum` (b2d_set_sins_impl(3))
// also spec_allpass | spec_noise
struct SinsWorkspace { size_t sinus, ir_ap, ir_n, spec_ap, spec_n, bytes; };
inline SinsWorkspace sins_workspace(int B, int nF, int block, int n_mag_allpass, int n_mag_noise, bool spectrum) {
    SinsWorkspace w{};
    if (B <= 0 || nF <= 0 || block <= 0 || n_mag_allpass < 2 || n_mag_noise < 2) return w;
    const size_t T = (size_t)B * nF * block, F = (size_t)B * nF;
    w.sinus = ws_append(w.bytes, T);
    w.ir_ap = ws_append(w.bytes, F * 2 * (n_mag_allpass - 1));
    w.ir_n = ws_append(w.bytes, F * 2 * (n_mag_noise - 1));
    if (spectrum) {
        w.spec_ap = ws_append(w.bytes, fir_spec_floats(B, nF));
        w.spec_n = ws_append(w.bytes, fir_spec_floats(B, nF));
    }
    return w;
}
// comb [B, T] | allpassed [B, T] | noise [B, T] | ir_allpass | ir_harmonic | ir_noise [B, nF, 2 (M - 1)]
struct CombSubWorkspace { size_t comb, allpassed, noise, ir_ap, ir_h, ir_n, bytes; };
inline CombSubWorkspace combsub_workspace(int B, int nF, int block, int n_mag_allpass, int n_mag_harmonic,
                                          int n_mag_noise) {
    CombSubWorkspace w{};
    if (B <= 0 || nF <= 0 || block <= 0 || n_mag_allpass < 2 || n_mag_harmonic < 2 || n_mag_noise < 2) return w;
    const size_t T = (size_t)B * nF * block, F = (size_t)B * nF;
    w.comb = ws_append(w.bytes, T);
    w.allpassed = ws_append(w.bytes, T);
    w.noise = ws_append(w.bytes, T);
    w.ir_ap = ws_append(w.bytes, F * 2 * (n_mag_allpass - 1));
    w.ir_h = ws_append(w.bytes, F * 2 * (n_mag_harmonic - 1));
    w.ir_n = ws_append(w.bytes, F * 2 * (n_mag_noise - 1));
    return w;
}

}  // namespace b2d

// ---------------------------------------------------------------------------------------
// device side
// ---------------------------------------------------------------------------------------
#define B2D_PI_F 3.14159265358979323846f
#define B2D_TWO_PI_F 6.28318530717958647692f

namespace b2d {

// Philox4x32-R (Salmon et al. 2011).  counter = (c0,c1,c2,c3), key = (k0,k1).  R = 10 is the standard generator (what
// torch / cuRAND use); R = 7 is the smallest round count the paper reports as passing BigCrush ("Crush-resistant") and is
// offered for the noise of the excitation generator only, where the generator is 57 % of the kernel's instructions.
template <int ROUNDS>
__device__ __forceinline__ uint4 philox4x32(uint4 c, uint2 k) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < ROUNDS; ++r) {
        uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
        uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += W0;
        k.y += W1;
    }
    return c;
}

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) { return philox4x32<10>(c, k); }

// 4 uniforms in [-1, 1) for samples 4*quad .. 4*quad+3 of utterance `utt`.
// Same 24-bit construction as torch.rand (x * 2^-24), then *2-1 (ddsp/vocoder.py:603).
__device__ __forceinline__ float4 philox_uniform_pm1(uint64_t seed, uint64_t utt, uint32_t quad) {
    uint4 r = philox4x32_10(make_uint4(quad, 0u, (uint32_t)utt, (uint32_t)(utt >> 32)),
                            make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
    const float s = 1.0f / 8388608.0f;  // 2^-23: (x>>8)*2^-24*2 - 1
    return make_float4((float)(r.x >> 8) * s - 1.0f, (float)(r.y >> 8) * s - 1.0f,
                       (float)(r.z >> 8) * s - 1.0f, (float)(r.w >> 8) * s - 1.0f);
}

// --- mbarrier + 1-D bulk async copy (TMA, SASS: UBLKCP) ---------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// global -> shared, `bytes` multiple of 16, both addresses 16-byte aligned.
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gmem_src, uint32_t bytes,
                                            uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(smem_dst)),
        "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}

__device__ __forceinline__ void st_global_v4(float* p, float4 v) {
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x),
                 "f"(v.y), "f"(v.z), "f"(v.w)
                 : "memory");
}

}  // namespace b2d
