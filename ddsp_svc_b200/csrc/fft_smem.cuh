// N-point complex FFT (N = 1024, 2048 or 4096) in shared memory for a 128-thread CTA: three in-place Stockham passes
// (radix 16, R2, 8 with R2 = N/128) over NBATCH independent transforms stored back to back, data padded by one slot
// per 16 so every pass is bank-conflict free.  Used by combsubfast.cu (N = 1024), ltv_fir_fft.cu, superfast.cu and
// mel.cu (1024 / 2048) and rss_loss.cu (all three: the Bluestein transforms).
// Index formulas pinned by tests/test_csfast_math.py and by the host emulation of both kernels (tests/emu/).
#pragma once
#include "fft_regs.cuh"

namespace b2d_fft_smem {
using namespace b2d_fft;

constexpr int kThreads = 128;

__device__ __forceinline__ int padi(int i) { return i + (i >> 4); }   // one pad slot per 16: conflict-free passes

template <int N> struct Plan {
    static_assert(N == 1024 || N == 2048 || N == 4096, "supported sizes");
    static constexpr int kN = N;
    static constexpr int kPad = N + N / 16;          // complex slots of one padded FFT buffer
    static constexpr int kR2 = N / 128;              // radix of the middle pass: 8, 16 or 32 (N = 1024, 2048, 4096)
    static constexpr int kTw2 = (kR2 - 1) * 16;      // exp(-2 pi i r k / (16 R2)), r = 1..R2-1, k < 16
    static constexpr int kTw3 = N / 8;               // exp(-2 pi i k / N), k < N/8
};

// One radix-R Stockham pass over NBATCH independent N-point FFTs stored back to back (FFT g at buf + g*kPad),
// in place.
//   butterfly j: v[r] = in[j + r N/R] * exp(-2 pi i r (j % NS) / (NS R));  DFT_R;  out[(j/NS) NS R + j%NS + r NS] = v[r]
// TW: 0 none (NS = 1), 1 full table tw[(r-1) NS + k], 2 powers of tw[k] = exp(-2 pi i k / (NS R))
// The batch is processed in stages that each cover WHOLE transforms: 128 butterflies when a transform has at most 128
// of them (one or two transforms per stage, one butterfly per thread), or one transform with N/R/128 butterflies per
// thread otherwise.  A stage reads, hits a barrier, then writes; different stages touch different transforms, so stage
// s+1 may start reading while other threads still write stage s, and only one stage's butterflies are live per thread.
// Barriers per pass: stages + 1.
// ZU (first pass only: R = 16, NS = 1): the upper half of every transform is zero padding and is neither read nor
// required to be initialised -- half the loads, no zero fill, pruned butterfly (Dft16ZeroUpper).
template <int N, int R, int NS, int TW, int NBATCH, bool PK = false, bool ZU = false>
__device__ __forceinline__ void fft_pass(float2* buf, const float2* __restrict__ tw, int tid) {
    static_assert(!ZU || (R == 16 && NS == 1 && TW == 0), "zero-upper pruning applies to the first radix-16 pass");
    constexpr int NB = N / R;                                        // butterflies per FFT
    constexpr int PER = NB > kThreads ? NB / kThreads : 1;           // butterflies per thread and stage
    constexpr int FPS = NB >= kThreads ? 1 : kThreads / NB;          // FFTs per stage
    constexpr int STAGES = (NBATCH + FPS - 1) / FPS;
    constexpr int kPad = Plan<N>::kPad;
    static_assert(NB % kThreads == 0 || kThreads % NB == 0, "a stage must hold whole FFTs");
#pragma unroll
    for (int s = 0; s < STAGES; ++s) {
        float2 v[PER][R];
        int gidx[PER], jidx[PER];
        bool active[PER];
#pragma unroll
        for (int u = 0; u < PER; ++u) {
            const int idx = tid + u * kThreads;                      // butterfly index inside the stage
            const int g = s * FPS + idx / NB, j = idx % NB, k = j % NS;
            gidx[u] = g; jidx[u] = j; active[u] = g < NBATCH;
            if (active[u]) {
                const float2* fft = buf + g * kPad;
#pragma unroll
                for (int r = 0; r < (ZU ? R / 2 : R); ++r) v[u][r] = fft[padi(j + r * NB)];
                if (TW == 1) {
#pragma unroll
                    for (int r = 1; r < R; ++r) v[u][r] = cmul(v[u][r], tw[(r - 1) * NS + k]);
                } else if (TW == 2) {
                    const float2 w1 = tw[k];
                    const float2 w2 = cmul(w1, w1), w3 = cmul(w2, w1), w4 = cmul(w2, w2);
                    const float2 w5 = cmul(w4, w1), w6 = cmul(w4, w2), w7 = cmul(w4, w3);
                    v[u][1] = cmul(v[u][1], w1); v[u][2] = cmul(v[u][2], w2); v[u][3] = cmul(v[u][3], w3);
                    v[u][4] = cmul(v[u][4], w4); v[u][5] = cmul(v[u][5], w5); v[u][6] = cmul(v[u][6], w6);
                    v[u][7] = cmul(v[u][7], w7);
                }
                if (ZU) Dft16ZeroUpper<PK>::run(v[u]);
                else Dft<R, PK>::run(v[u]);
            }
        }
        __syncthreads();
#pragma unroll
        for (int u = 0; u < PER; ++u) {
            if (active[u]) {
                float2* fft = buf + gidx[u] * kPad;
                const int j = jidx[u];
                const int base = (j / NS) * NS * R + (j % NS);
#pragma unroll
                for (int r = 0; r < R; ++r) fft[padi(base + r * NS)] = v[u][r];
            }
        }
    }
    __syncthreads();
}

// forward FFT of NBATCH transforms at buf, buf + kPad, ...
template <int N, int NBATCH, bool PK = false, bool ZU = false>
__device__ __forceinline__ void fft_forward(float2* buf, const float2* tw2, const float2* tw3, int tid) {
    constexpr int R2 = Plan<N>::kR2;
    fft_pass<N, 16, 1, 0, NBATCH, PK, ZU>(buf, nullptr, tid);
    fft_pass<N, R2, 16, 1, NBATCH, PK>(buf, tw2, tid);
    fft_pass<N, 8, 16 * R2, 2, NBATCH, PK>(buf, tw3, tid);
}

// twiddle tables of passes 2 and 3 (call with all threads, then __syncthreads)
template <int N>
__device__ __forceinline__ void init_twiddles(float2* tw2, float2* tw3, int tid) {
    constexpr int R2 = Plan<N>::kR2;
    for (int i = tid; i < Plan<N>::kTw2; i += kThreads) {
        const int r = i / 16 + 1, k = i % 16;
        float sn, cs; sincospif(-2.0f * (float)(r * k) / (float)(16 * R2), &sn, &cs);
        tw2[i] = make_float2(cs, sn);
    }
    for (int i = tid; i < Plan<N>::kTw3; i += kThreads) {
        float sn, cs; sincospif(-2.0f * (float)i / (float)N, &sn, &cs);
        tw3[i] = make_float2(cs, sn);
    }
}

}  // namespace b2d_fft_smem
