// Bluestein's chirp z-transform on the shared-memory Stockham FFT of fft_smem.cuh: an n-point DFT of any length n (primes
// included) as a cyclic convolution of size M = 1024 / 2048 / 4096.  Used by rss_loss.cu (all n outputs of n in
// [256, 2047]) and mel.cu (the first K bins of the keyshifted n' in [hop, 3072]).
//
//   X[k] = conj(c[k]) * (u (*) h)[k],   u[m] = z[m] conj(c[m]) (m < n, zero to M),   c[m] = exp(+i pi (m^2 mod 2n) / n)
//   h    = c on [0, n_out) and its mirror c[M - m] on (M - n, M);  u (*) h = IFFT_M(FFT_M(u) * FFT_M(h))
//
// The convolution gives bins k < n_out without wrap-around when M >= n + n_out - 1 (bluestein_size).  FFT_M(h) / M and
// the chirp come from a per-n table built on the host in float64 (rounded once to fp32); the inverse FFT is a forward
// FFT read at (M - k) mod M.
//
// Per-n table (floats): [0, kWinOff) caller-defined scalars; the window (n floats) at kWinOff; the chirp (n float2) at
// chirp_off(n); FFT_M(h) / M (M float2) at hspec_off(n).  bluestein_table_floats(n, n_out) floats in all.
#pragma once
#include "fft_smem.cuh"

namespace b2d_bluestein {
using namespace b2d_fft;
using b2d_fft_smem::kThreads;
using b2d_fft_smem::padi;

constexpr int kWinOff = 4;
__host__ __device__ __forceinline__ int chirp_off(int n) { return kWinOff + ((n + 3) & ~3); }
__host__ __device__ __forceinline__ int hspec_off(int n) { return chirp_off(n) + 2 * n; }
// the transform size for bins [0, n_out) of an n-point DFT: the smallest of 1024 / 2048 / 4096 that is >= n + n_out - 1
// (0: none is large enough)
__host__ __device__ __forceinline__ int bluestein_size(int n, int n_out) {
    const int need = n + n_out - 1;
    return need <= 1024 ? 1024 : need <= 2048 ? 2048 : need <= 4096 ? 4096 : 0;
}
__host__ __device__ __forceinline__ int bluestein_table_floats(int n, int n_out) {
    return hspec_off(n) + 2 * bluestein_size(n, n_out);
}

// Bluestein's DFT_n of the NB transforms at z0 (, z0 + kPad): on entry slot m < n holds z[m] conj(c[m]) and [n, M) is
// zero; on exit DFT_n(z)[k] = conj(c[k]) z[(M - k) mod M]  (read with bluestein_out).  ZU (n <= M / 2): the first FFT
// skips the zero upper half, which then need not be written.
template <int M, int NB, bool ZU = true>
__device__ __forceinline__ void bluestein_core(float2* z0, const float2* __restrict__ hspec, const float2* tw2,
                                               const float2* tw3, int tid) {
    constexpr int kPad = b2d_fft_smem::Plan<M>::kPad;
    b2d_fft_smem::fft_forward<M, NB, true, ZU>(z0, tw2, tw3, tid);
    for (int i = tid; i < M; i += kThreads) {
        const float2 h = __ldg(hspec + i);
        z0[padi(i)] = cmul(z0[padi(i)], h);
        if (NB == 2) z0[kPad + padi(i)] = cmul(z0[kPad + padi(i)], h);
    }
    __syncthreads();
    b2d_fft_smem::fft_forward<M, NB, true>(z0, tw2, tw3, tid);
}

template <int M>
__device__ __forceinline__ float2 bluestein_out(const float2* z, const float2* __restrict__ chirp, int k) {
    const float2 c = __ldg(chirp + k), v = z[padi((M - k) & (M - 1))];
    return make_float2(fmaf(c.x, v.x, c.y * v.y), fmaf(c.x, v.y, -c.y * v.x));      // conj(c) v
}

}  // namespace b2d_bluestein
