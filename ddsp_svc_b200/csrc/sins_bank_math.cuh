// Arithmetic of the additive sinusoid bank shared by sins_bank.cu (stand-alone kernel) and ltv_fir_fft.cu (bank fused
// into the FFT-domain FIR kernel): harmonic factoring h = a + 16 b, paired (register-pair) accumulation.  See sins_bank.cu for the
// derivation; reference ddsp/vocoder.py:580,585-594.
#pragma once
#ifndef B2D_HOST_EMU               // tests/emu/ runs sins_bwd.cu on the CPU: only the asm-free helpers below exist there
#include "b2d_common.cuh"
#endif

// 1 (default): even anchors by double-angle chains (halves the SFU
// work of the anchors); 0: every anchor by __sincosf (round-1 code)
#ifndef B2D_BANK_DOUBLE_ANGLE
#define B2D_BANK_DOUBLE_ANGLE 1
#endif

namespace b2d_bank {

constexpr int kGroup = 128;  // harmonics per group = 16 anchors x 8 bases
constexpr int kNA = 16;      // anchors
constexpr int kNBmax = 8;    // bases per group

struct BankParams {
    const float* f0;
    const double* frame_phase;
    const float* c_amp;
    long long ctrl_stride;
    int nF, P, H;
    double inv_sr;
    float nyquist;
    int round_fp32;
    int use_tma;
    float* out;
};

// slot of 0-based harmonic index hh inside a padded row: [group][anchor][base]
__device__ __forceinline__ int slot_of(int hh) {
    int g = hh >> 7, r = hh & 127;
    return (g << 7) + ((r & (kNA - 1)) * kNBmax) + (r / kNA);
}

#ifndef B2D_HOST_EMU
typedef unsigned long long u64;
__device__ __forceinline__ u64 pack2(float lo, float hi) { u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ void unpack2(u64 v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
// lane-wise fma of two register pairs (Hopper has no packed FP32 FMA: two FFMAs, same roundings)
__device__ __forceinline__ u64 ffma2(u64 a, u64 b, u64 c) {
    float a0, a1, b0, b1, c0, c1;
    unpack2(a, a0, a1); unpack2(b, b0, b1); unpack2(c, c0, c1);
    return pack2(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}

// One group of (up to) 128 harmonics for 4 samples.  NB = bases actually present (1..8).
// The amplitudes of two neighbouring bases are interpolated as one register pair, and (P_b, Q_b) += (sin, cos) * amp
// is one pair update.
template <int NB, bool TRIVIAL0>
__device__ __forceinline__ void bank_group(const float* __restrict__ arow, const float* __restrict__ drow,
                                           int group, const float (&x32)[4], const float (&phase)[4],
                                           const float (&frac)[4], float (&acc)[4]) {
    constexpr int NP = (NB + 1) / 2;          // base pairs
    u64 PQ[4][2 * NP];
#pragma unroll
    for (int s = 0; s < 4; ++s)
#pragma unroll
        for (int b = 0; b < 2 * NP; ++b) PQ[s][b] = 0ull;

    const float4* a4 = reinterpret_cast<const float4*>(arow + group * kGroup);
    const float4* d4 = reinterpret_cast<const float4*>(drow + group * kGroup);
    const float hbase = (float)(group * kGroup);

#if B2D_BANK_DOUBLE_ANGLE
    // Anchors in chains 1-2-4-8-16 | 3-6-12 | 5-10 | 7-14 | 9 | 11 | 13 | 15: only the odd anchors call the SFU (16 MUFU per
    // sample instead of 32); an even anchor comes from its half by the double-angle identities sin 2x = 2 s c,
    // cos 2x = 1 - 2 s^2 (3 FP32 operations).  The chain keeps ONE (sin, cos) pair per sample alive.  Error: each doubling
    // doubles the absolute error of the pair; anchor 16 (four doublings from an argument in [-pi, pi], where the SFU is
    // most accurate) carries ~16 x 2^-22, the same order as MUFU.SIN on the unreduced argument 16 phi it replaces.
    constexpr int kOrder[kNA] = {0, 1, 3, 7, 15, 2, 5, 11, 4, 9, 6, 13, 8, 10, 12, 14};      // anchor index a - 1
    constexpr bool kFresh[kNA] = {true, false, false, false, false, true, false, false, true, false, true, false, true, true, true, true};
    float sa[4], ca[4];
#pragma unroll
    for (int i = 0; i < kNA; ++i) {
        const int a = kOrder[i];
#else
#pragma unroll 2
    for (int a = 0; a < kNA; ++a) {
#endif
        u64 Ap[4], Dp[4];
        {
            const float4 A0 = a4[2 * a], D0 = d4[2 * a];
            Ap[0] = pack2(A0.x, A0.y); Ap[1] = pack2(A0.z, A0.w);
            Dp[0] = pack2(D0.x, D0.y); Dp[1] = pack2(D0.z, D0.w);
            if (NB > 4) {
                const float4 A1 = a4[2 * a + 1], D1 = d4[2 * a + 1];
                Ap[2] = pack2(A1.x, A1.y); Ap[3] = pack2(A1.z, A1.w);
                Dp[2] = pack2(D1.x, D1.y); Dp[3] = pack2(D1.z, D1.w);
            }
        }
        const float af = (float)(a + 1);
#pragma unroll
        for (int s = 0; s < 4; ++s) {
#if B2D_BANK_DOUBLE_ANGLE
            if (kFresh[i]) {
                __sincosf(af * phase[s], &sa[s], &ca[s]);
            } else {
                const float so = sa[s], co = ca[s];
                sa[s] = (2.0f * so) * co;
                ca[s] = fmaf(-2.0f * so, so, 1.0f);
            }
            const u64 sc = pack2(sa[s], ca[s]), fr = pack2(frac[s], frac[s]);
#else
            float sa, ca;
            __sincosf(af * phase[s], &sa, &ca);
            const u64 sc = pack2(sa, ca), fr = pack2(frac[s], frac[s]);
#endif
#pragma unroll
            for (int bp = 0; bp < NP; ++bp) {
                float amp0, amp1;
                unpack2(ffma2(Dp[bp], fr, Ap[bp]), amp0, amp1);        // amplitudes of bases 2bp, 2bp+1
                PQ[s][2 * bp] = ffma2(sc, pack2(amp0, amp0), PQ[s][2 * bp]);
                if (2 * bp + 1 < NB) PQ[s][2 * bp + 1] = ffma2(sc, pack2(amp1, amp1), PQ[s][2 * bp + 1]);
            }
        }
    }
    // rotate each base by (hbase + 16 b) * phase; the rotation angle is reduced exactly in
    // cycles (fma) before the SFU call because it reaches ~100 revolutions.
#pragma unroll
    for (int s = 0; s < 4; ++s) {
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            float Pv, Qv;
            unpack2(PQ[s][b], Pv, Qv);
            if (TRIVIAL0 && b == 0) {
                acc[s] += Pv;
            } else {
                const float hb = hbase + (float)(kNA * b);
                const float n = rintf(hb * x32[s]);
                const float r = fmaf(hb, x32[s], -n);
                float so, co;
                __sincosf(B2D_TWO_PI_F * r, &so, &co);
                acc[s] = fmaf(Pv, co, acc[s]);
                acc[s] = fmaf(Qv, so, acc[s]);
            }
        }
    }
}
#endif  // B2D_HOST_EMU


// activated amplitude of 0-based harmonic hh at a frame with pitch f0:  exp(c)/128 * (1[f0 (hh+1) < sr/2] + 1e-7)
// (ddsp/vocoder.py:580,585, ddsp/core.py:73-77)
__device__ __forceinline__ float activate_amp(float c, float f0, int hh, float nyquist) {
    const float keep = ((f0 * (float)(hh + 1)) < nyquist ? 1.0f : 0.0f) + 1e-7f;
    return (expf(c) * 0.0078125f) * keep;
}

// wrapped phase (cycles, fp32) of sample j of a frame: S + ((j+1) fk + dk j (j+1) / (2P)) / sr in fp64, rounded where
// the reference rounds (ddsp/vocoder.py:566-572)
__device__ __forceinline__ float sample_phase(double S, double fk, double dk, int j, double inv2P, double inv_sr, int round_fp32) {
    const double jj = (double)j;
    double x = S + ((jj + 1.0) * fk + dk * (jj * (jj + 1.0)) * inv2P) * inv_sr;
    if (round_fp32) x = (double)(float)x;
    x -= rint(x);
    return (float)x;
}

}  // namespace b2d_bank
