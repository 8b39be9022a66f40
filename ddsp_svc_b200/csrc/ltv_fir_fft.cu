// K4f: linear time-varying FIR evaluated in the FFT domain (alternative to the direct-form kernels of ltv_fir.cu).
// Same contract as b2d::ltv_fir_launch (reference ddsp/core.py:120-182):
//
//   y[n] = sum_tau ((1-phi_m) h_f[tau] + phi_m h_{f+1}[tau]) x[m],   m = n + L/2 - tau, f = floor(m/P), phi_m = (m mod P)/P
//
// Regrouped by INPUT hop g (samples m = gP + i, i < P):   y = sum_g  x_g * h_g  +  (phi x_g) * (h_{g+1} - h_g)
// -- two linear convolutions of a P-sample segment with L taps, which an N-point FFT holds without wrap-around when
// P + L - 1 <= N: N = 1024 for L <= 512 (Sins, CombSub's all-pass and noise filters), N = 2048 for L <= 1024 (CombSub's
// 1022-tap harmonic filter).  A CTA walks the input hops of its chunk TWO at a time; per pair and job:
//   * x_g and phi*x_g are real: one complex FFT of (x_g + j phi x_g) gives both spectra (split by conjugate
//     symmetry); the impulse responses of frames g+1 and g+2 share one FFT the same way (frame g's spectrum is kept
//     in registers from the previous pair);
//   * Y_g = X_g H_g + XU_g (H_{g+1} - H_g) and Y_{g+1} likewise are spectra of real segments: one inverse FFT of
//     Y_g + j Y_{g+1} returns both.  Only signals of the SAME job are ever paired in one transform, so the fp32
//     round-off of a loud channel (harmonic) never leaks into a quiet one (filtered noise);
//   * all forward transforms of a pair (2 inputs + 1 impulse-response pair per job) run as one batch through the
//     shared-memory Stockham passes of fft_smem.cuh, then all inverse transforms as a second batch;
//   * every 1021-sample output segment is overlap-added into a 4-hop ring per job at its delay-compensated position;
//     a hop is complete once the segment of the FOLLOWING input hop has been added and is then written exactly once
//     (y1, y2 and mix = y1 + y2 (+ addend)) with 128-bit stores -- deterministic, no atomics.
// 4 FFT-1024 per hop and job pair replace 2 x 2 x L x P = 1.04 M FMAs of the direct form (L = 510): ~4x fewer
// instructions.  A CTA owns G hops (G even) of one utterance and processes the G+2 input hops that reach them (they
// form whole pairs); white-noise input (x2 == nullptr) is the same Philox stream as in the direct-form kernels.
//
// This is the automatic dispatch for block size 512 and <= 1024 taps (ltv_fir.cu).  Logic additionally pinned on the CPU by
// the host emulation in tests/emu/ (tests/test_emu_ltv_fir_fft.py, race check in tests/test_emu_tsan.py).
#ifndef B2D_HOST_EMU
#include "b2d_common.cuh"
#include "sins_bank_math.cuh"
#endif
#include "fft_smem.cuh"

using namespace b2d_fft_smem;

namespace {

constexpr int kHop = 512;
constexpr int kRing = 4 * kHop;          // power of two: slot = (t - t_lo) & (kRing - 1)

struct FftFirJob {
    const float* x;    // [B, T] or nullptr -> in-kernel uniform noise
    const float* ir;   // [B, nF, L] impulse responses; SPEC variant: [B, nF, N/2] float2 packed spectra (ir_spectrum_kernel)
    float* y;          // [B, T] or nullptr
    int L;
};

// BANK variant (Sins): job 0's input is not read from memory but synthesised in the kernel -- the additive sinusoid bank
// of the hop (sins_bank_math.cuh, the arithmetic of sins_bank.cu) is evaluated straight into the FFT buffer.  The FIR
// kernel alone is latency bound (barriers, shared-memory round trips: ~54 % issue slots used, FMA pipe 37 %) and the bank
// alone is FMA / SFU bound; in one kernel the warps of the three resident CTAs sit in different phases, so the bank's
// arithmetic fills the issue slots the transforms leave empty, the [B, T] sinusoid tensor never exists (113 MB of HBM
// traffic) and a launch disappears.
struct FftFirBank {
    const float* f0;             // [B, nF]
    const double* frame_phase;   // [B, nF] unwrapped cycles at frame starts (phase_scan.cu)
    const float* c_amp;          // raw amplitudes, frame stride ctrl_stride
    long long ctrl_stride;
    int H;
    double inv_sr;
    float nyquist;
    int round_fp32;
};

struct FftFirParams {
    FftFirJob job[2];
    const float* addend;
    float* mix;
    unsigned long long seed;
    long long utt_off;
    int nF, G;
    FftFirBank bank;
};

constexpr int kBankRow = 128;            // harmonics per activated amplitude row of the BANK variant (H <= 128)
// SPEC variant: the spectra of the impulse responses are read from memory (ir_spectrum_kernel made them once per frame),
// so the HH buffers and a quarter of the transforms disappear: 2 NJ buffers -> 53.4 KB for N = 1024, NJ = 2 -> 4 CTAs per SM
template <int N, int NJ, int NBANK = 0, bool SPEC = false> constexpr size_t fir_fft_smem() {
    return (size_t)(SPEC ? 2 : 3) * NJ * Plan<N>::kPad * sizeof(float2) + (size_t)(Plan<N>::kTw2 + Plan<N>::kTw3) * sizeof(float2) +
           (size_t)NJ * kRing * sizeof(float) + (NBANK ? (size_t)5 * kBankRow * sizeof(float) : 0);
}   // N = 1024: NJ = 2 -> 70528 B (3 CTAs per SM), NJ = 1 -> 36224 B;  N = 2048: NJ = 1 -> 64384 B, NJ = 2 -> 124800 B

// spectra of two real sequences a, c from Z = FFT(a + j c):  A[k] = (Z[k] + conj Z[N-k]) / 2,  C[k] = (Z[k] - conj Z[N-k]) / 2j
__device__ __forceinline__ void split2(float2 zk, float2 zm, float2& A, float2& C) {
    A = make_float2(0.5f * (zk.x + zm.x), 0.5f * (zk.y - zm.y));
    C = make_float2(0.5f * (zk.y + zm.y), 0.5f * (zm.x - zk.x));
}

// PK: the "packed" complex-addition policy (fft_regs.cuh Ar<true>; scalar on Hopper)
// NBANK: 0 = inputs from memory / Philox; 4 or 8 = job 0 is the sinusoid bank with that many bases of 16 harmonics
// SPEC: job[j].ir holds the packed 1024-point spectra of the impulse responses instead of the taps
template <int N, int NJ, bool PK, int NBANK = 0, bool SPEC = false>
__global__ void __launch_bounds__(kThreads, (N == 2048 && NJ == 2) ? 1 : (SPEC ? 4 : 3)) ltv_fir_fft_kernel(FftFirParams p) {
    constexpr int kN = N, kPad = Plan<N>::kPad, kTw2 = Plan<N>::kTw2, kTw3 = Plan<N>::kTw3;
    constexpr int kBins = N / 2 / kThreads;          // bins k = tid + 128 u per thread (DC.. N/2-1); Nyquist on thread 0
    extern __shared__ __align__(16) unsigned char smem_raw[];
    // buffer b of the batch lives at F + b * kPad:  XA(j) = j  (hop g; later the paired output of job j),
    // XB(j) = NJ + j (hop g+1),  HH(j) = 2 NJ + j (impulse responses of frames g+1 and g+2)
    float2* F = reinterpret_cast<float2*>(smem_raw);
    float2* tw2 = F + (SPEC ? 2 : 3) * NJ * kPad;
    float2* tw3 = tw2 + kTw2;
    float* ring = reinterpret_cast<float*>(tw3 + kTw3);          // [NJ][kRing]
    float* bank_act = ring + NJ * kRing;                         // BANK: [3][128] activated amplitudes of frames g, g+1, g+2
    float* bank_dlt = bank_act + 3 * kBankRow;                   //       [2][128] their differences

    const int tid = threadIdx.x;
    const int b = blockIdx.y;
    const int nF = p.nF, T = nF * kHop;
    const int h0 = blockIdx.x * p.G, h1 = min(h0 + p.G, nF);
    const int t_lo = h0 * kHop, t_hi = h1 * kHop;
    const unsigned long long utt = (unsigned long long)(p.utt_off + b);

    init_twiddles<N>(tw2, tw3, tid);
    for (int i = tid; i < NJ * kRing; i += kThreads) ring[i] = 0.f;

    // (h_j[fa], h_j[fb]) as one complex sequence, zero-padded to 1024; frame indices clamp (h_{nF} := h_{nF-1})
    auto load_ir_pair = [&](int j, int fa, int fb, bool with_b) {
        const int L = p.job[j].L;
        const float* base = p.job[j].ir + (size_t)b * nF * L;
        const float* ra = base + (size_t)min(max(fa, 0), nF - 1) * L;
        const float* rb = base + (size_t)min(max(fb, 0), nF - 1) * L;
        float2* buf = F + (2 * NJ + j) * kPad;
        // taps L <= N/2: only the lower half of the buffer is written, the transform treats the upper half as zeros
#pragma unroll
        for (int u = 0; u < kN / 2 / kThreads; ++u) {
            const int tau = tid + u * kThreads;
            const bool in = tau < L;
            buf[padi(tau)] = make_float2(in ? __ldg(ra + tau) : 0.f, (in && with_b) ? __ldg(rb + tau) : 0.f);
        }
    };
    // Global loads of a hop pair (input samples read from memory, impulse-response taps), issued ONE ITERATION AHEAD into
    // registers: they are in flight during the previous pair's transforms instead of stalling the head of the iteration.
    constexpr int kTau = kN / 2 / kThreads;
    struct Prefetch { float4 xa[NJ], xb[NJ]; float ha[NJ][kTau], hb[NJ][kTau]; };
    auto fetch = [&](int g, Prefetch& q) {
        const bool a_ok = g >= 0, b_ok = g + 1 <= nF - 1;
        const int i0 = tid << 2;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            q.xa[j] = q.xb[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p.job[j].x && !(NBANK && j == 0)) {
                const float* xr = p.job[j].x + (size_t)b * T + i0;
                if (a_ok) q.xa[j] = __ldg(reinterpret_cast<const float4*>(xr + (size_t)g * kHop));
                if (b_ok) q.xb[j] = __ldg(reinterpret_cast<const float4*>(xr + (size_t)(g + 1) * kHop));
            }
            if (!SPEC) {
                const int L = p.job[j].L;
                const float* base = p.job[j].ir + (size_t)b * nF * L;
                const float* ra = base + (size_t)min(max(g + 1, 0), nF - 1) * L;
                const float* rb = base + (size_t)min(max(g + 2, 0), nF - 1) * L;
#pragma unroll
                for (int u = 0; u < kTau; ++u) {
                    const int tau = tid + u * kThreads;
                    q.ha[j][u] = tau < L ? __ldg(ra + tau) : 0.f;
                    q.hb[j][u] = tau < L ? __ldg(rb + tau) : 0.f;
                }
            }
        }
    };
    auto put_ir_pair = [&](int j, const Prefetch& q) {
        float2* buf = F + (2 * NJ + j) * kPad;
#pragma unroll
        for (int u = 0; u < kTau; ++u) buf[padi(tid + u * kThreads)] = make_float2(q.ha[j][u], q.hb[j][u]);
    };
    // x_j[gP + i] (1 + j i/P) for i < P, zeros above; `present` false -> all zeros (hop outside the chunk's reach);
    // `pre` = the hop's samples when the job reads its input from memory (prefetched), else Philox noise is drawn here
    auto load_x = [&](int j, int g, bool present, float4 pre, float2* buf) {
        const int i0 = tid << 2;
        const int m0 = g * kHop + i0;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (present) {
            if (p.job[j].x) v = pre;
            else v = b2d::philox_uniform_pm1(p.seed, utt, (uint32_t)(m0 >> 2));
        }
        const float s = 1.0f / kHop;
        buf[padi(i0 + 0)] = make_float2(v.x, v.x * ((float)(i0 + 0) * s));
        buf[padi(i0 + 1)] = make_float2(v.y, v.y * ((float)(i0 + 1) * s));
        buf[padi(i0 + 2)] = make_float2(v.z, v.z * ((float)(i0 + 2) * s));
        buf[padi(i0 + 3)] = make_float2(v.w, v.w * ((float)(i0 + 3) * s));
#pragma unroll
        for (int z = kHop; z < kN / 2; z += kHop)          // (N = 2048 only) zeros up to N/2; the upper half is implicit
#pragma unroll
            for (int e = 0; e < 4; ++e) buf[padi(z + i0 + e)] = make_float2(0.f, 0.f);
    };

#ifndef B2D_HOST_EMU
    // BANK: the 4 samples i0..i0+3 of hop g of the sinusoid bank (amplitude rows r, r+1 of bank_act) -> (x, phi x)
    auto bank_x = [&](int g, int r, bool present, float2* buf) {
        const int i0 = tid << 2;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        if (NBANK && present) {
            const float* f0row = p.bank.f0 + (size_t)b * nF;
            const double fk = (double)__ldg(f0row + g), dk = (double)__ldg(f0row + min(g + 1, nF - 1)) - fk;
            const double S = __ldg(p.bank.frame_phase + (size_t)b * nF + g);
            float x32[4], phase[4], frac[4];
#pragma unroll
            for (int s = 0; s < 4; ++s) {
                x32[s] = b2d_bank::sample_phase(S, fk, dk, i0 + s, 0.5 / (double)kHop, p.bank.inv_sr, p.bank.round_fp32);
                phase[s] = x32[s] * B2D_TWO_PI_F;
                frac[s] = (float)(i0 + s) * (1.0f / kHop);
            }
            b2d_bank::bank_group<(NBANK ? NBANK : 1), true>(bank_act + r * kBankRow, bank_dlt + r * kBankRow, 0, x32, phase, frac, acc);
        }
        const float s = 1.0f / kHop;
#pragma unroll
        for (int e = 0; e < 4; ++e) buf[padi(i0 + e)] = make_float2(acc[e], acc[e] * ((float)(i0 + e) * s));
#pragma unroll
        for (int z = kHop; z < kN / 2; z += kHop)
#pragma unroll
            for (int e = 0; e < 4; ++e) buf[padi(z + i0 + e)] = make_float2(0.f, 0.f);
    };
#endif

    // spectrum of frame g per job: bins k = tid + 128 u; thread 0 additionally holds DC (u = 0) and Nyquist (real)
    float2 Hp[NJ][kBins];
    float HpN[NJ];
    // Input hops are always transformed in the SAME pairs (2m-1, 2m), whatever the chunking: G is even, so the first hop
    // that reaches this chunk (h0 - 1, odd) starts a pair and the last one (h1, even) ends one -- no extra work, and
    // since the partner of a pair only enters through the round-off of the shared transforms, every output sample is
    // bit-identical for any G, batch split or shard.  Hop -1 (the partner of hop 0) does not exist: zeros.
    const int gs = h0 - 1, ge = min(h1, nF - 1);

    // SPEC: packed spectrum row of frame f (clamped) of job j: [0] = (DC, Nyquist), [k] = H[k] for k = 1 .. N/2-1
    auto spec_row = [&](int j, int f) -> const float2* {
        return reinterpret_cast<const float2*>(p.job[j].ir) + ((size_t)b * nF + min(max(f, 0), nF - 1)) * (kN / 2);
    };

    // ---- prologue: spectra of frame gs ----
    if (SPEC) {
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const float2* row = spec_row(j, gs);
#pragma unroll
            for (int u = 0; u < kBins; ++u) {
                const int k = tid + u * kThreads;
                const float2 h = __ldg(row + k);
                Hp[j][u] = k == 0 ? make_float2(h.x, 0.f) : h;
                if (k == 0) HpN[j] = h.y;
            }
        }
        __syncthreads();                                                // twiddles and the cleared rings
    } else {
#pragma unroll
        for (int j = 0; j < NJ; ++j) load_ir_pair(j, gs - 1, gs, true);    // exactly the (h_{g+1}, h_{g+2}) pair of hops gs-2, gs-1
        __syncthreads();
        fft_forward<N, NJ, PK, true>(F + 2 * NJ * kPad, tw2, tw3, tid);
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const float2* H = F + (2 * NJ + j) * kPad;
#pragma unroll
            for (int u = 0; u < kBins; ++u) {
                const int k = tid + u * kThreads;
                float2 unused;
                if (k == 0) Hp[j][u] = make_float2(H[padi(0)].y, 0.f);
                else split2(H[padi(k)], H[padi(kN - k)], unused, Hp[j][u]);
            }
            HpN[j] = H[padi(kN / 2)].y;                                 // only thread 0 uses it
        }
        __syncthreads();
    }

    // write hop h (complete) from the rings: y_j, mix; clear its ring slots
    auto emit = [&](int h) {
        const int slot = (((h - h0) * kHop) & (kRing - 1)) + (tid << 2);
        const size_t o = (size_t)b * T + (size_t)h * kHop + (tid << 2);
        float4 m = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            float4* r = reinterpret_cast<float4*>(ring + j * kRing + slot);
            const float4 v = *r;
            *r = make_float4(0.f, 0.f, 0.f, 0.f);
            if (p.job[j].y) b2d::st_global_v4(p.job[j].y + o, v);
            if (j == 0) m = v;
            else { m.x += v.x; m.y += v.y; m.z += v.z; m.w += v.w; }
        }
        if (p.mix) {
            if (p.addend) {
                const float4 a = __ldg(reinterpret_cast<const float4*>(p.addend + o));
                m.x += a.x; m.y += a.y; m.z += a.z; m.w += a.w;
            }
            b2d::st_global_v4(p.mix + o, m);
        }
    };

    Prefetch pf;
    fetch(gs, pf);
#pragma unroll 1
    for (int g = gs; g <= ge; g += 2) {
        const bool has_a = g >= 0, has_b = g + 1 <= nF - 1;      // properties of the utterance only, not of the chunking
        // ---- forward: both hops of every job and the impulse-response pairs as one batch ----
#ifndef B2D_HOST_EMU
        if (NBANK) {
            // activated amplitudes of frames g, g+1, g+2 (clamped: A[nF] := A[nF-1], ddsp/core.py:68) and their differences.
            // The rows were last read before the previous iteration's transform barriers.
#pragma unroll
            for (int r = 0; r < 3; ++r) {
                const int k = min(max(g + r, 0), nF - 1);
                float v = 0.f;
                if (tid < p.bank.H)
                    v = b2d_bank::activate_amp(__ldg(p.bank.c_amp + ((size_t)b * nF + k) * p.bank.ctrl_stride + tid),
                                               __ldg(p.bank.f0 + (size_t)b * nF + k), tid, p.bank.nyquist);
                bank_act[r * kBankRow + b2d_bank::slot_of(tid)] = v;
            }
            __syncthreads();
            bank_dlt[tid] = bank_act[kBankRow + tid] - bank_act[tid];
            bank_dlt[kBankRow + tid] = bank_act[2 * kBankRow + tid] - bank_act[kBankRow + tid];
            __syncthreads();
        }
#endif
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
#ifndef B2D_HOST_EMU
            if (NBANK && j == 0) {
                bank_x(g, 0, has_a, F + j * kPad);
                bank_x(g + 1, 1, has_b, F + (NJ + j) * kPad);
            } else
#endif
            {
                load_x(j, g, has_a, pf.xa[j], F + j * kPad);
                load_x(j, g + 1, has_b, pf.xb[j], F + (NJ + j) * kPad);
            }
            if (!SPEC) put_ir_pair(j, pf);
        }
        __syncthreads();
        if (g + 2 <= ge) fetch(g + 2, pf);                 // next pair's loads fly during this pair's transforms
        fft_forward<N, (SPEC ? 2 : 3) * NJ, PK, true>(F, tw2, tw3, tid);   // all have zero upper halves: pruned first pass

        // ---- Y_g = X_g H_g + XU_g (H_{g+1} - H_g),  Y_{g+1} = X_{g+1} H_{g+1} + XU_{g+1} (H_{g+2} - H_{g+1});
        //      paired as Y_g + j Y_{g+1} (Hermitian extension), stored re/im-swapped over XA(j) ----
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            float2* XA = F + j * kPad;
            const float2* XB = F + (NJ + j) * kPad;
            const float2* HH = F + (2 * NJ + j) * kPad;                 // (!SPEC)
            const float2* rowA = SPEC ? spec_row(j, g + 1) : nullptr;     // (SPEC) spectra of frames g+1, g+2
            const float2* rowB = SPEC ? spec_row(j, g + 2) : nullptr;
            float2 HaR[kBins], HbR[kBins];
            if (SPEC) {
#pragma unroll
                for (int u = 0; u < kBins; ++u) { HaR[u] = __ldg(rowA + tid + u * kThreads); HbR[u] = __ldg(rowB + tid + u * kThreads); }
            }
#pragma unroll
            for (int u = 0; u < kBins; ++u) {
                const int k = tid + u * kThreads;
                if (k == 0) continue;
                const int ik = padi(k), im = padi(kN - k);
                float2 Xa, XUa, Xb, XUb, Ha, Hb;
                split2(XA[ik], XA[im], Xa, XUa);
                split2(XB[ik], XB[im], Xb, XUb);
                if (SPEC) { Ha = HaR[u]; Hb = HbR[u]; }
                else split2(HH[ik], HH[im], Ha, Hb);
                const float2 ya = Ar<PK>::add(cmul(Xa, Hp[j][u]), cmul(XUa, Ar<PK>::sub(Ha, Hp[j][u])));
                const float2 yb = Ar<PK>::add(cmul(Xb, Ha), cmul(XUb, Ar<PK>::sub(Hb, Ha)));
                // Y[k] = ya + j yb;  Y[N-k] = conj(ya) + j conj(yb);  stored as (im, re)
                XA[ik] = make_float2(ya.y + yb.x, ya.x - yb.y);
                XA[im] = make_float2(yb.x - ya.y, ya.x + yb.y);
                Hp[j][u] = Hb;
            }
            if (tid == 0) {      // DC and Nyquist: every spectrum involved is real there
                const float2 a0 = XA[padi(0)], b0 = XB[padi(0)];                              // (X, XU), (X, XU)
                const float2 aN = XA[padi(kN / 2)], bN = XB[padi(kN / 2)];
                // (H_{g+1}, H_{g+2}) at DC and at Nyquist
                const float2 z0 = SPEC ? make_float2(HaR[0].x, HbR[0].x) : HH[padi(0)];
                const float2 zN = SPEC ? make_float2(HaR[0].y, HbR[0].y) : HH[padi(kN / 2)];
                const float hp0 = Hp[j][0].x, hpN = HpN[j];
                const float ya0 = fmaf(a0.y, z0.x - hp0, a0.x * hp0), yb0 = fmaf(b0.y, z0.y - z0.x, b0.x * z0.x);
                const float yaN = fmaf(aN.y, zN.x - hpN, aN.x * hpN), ybN = fmaf(bN.y, zN.y - zN.x, bN.x * zN.x);
                XA[padi(0)] = make_float2(yb0, ya0);
                XA[padi(kN / 2)] = make_float2(ybN, yaN);
                Hp[j][0] = make_float2(z0.y, 0.f);
                HpN[j] = zN.y;
            }
        }
        __syncthreads();

        // ---- inverse of the pairs (batch over jobs): hop g = stored .y / N, hop g+1 = stored .x / N ----
        fft_forward<N, NJ, PK>(F, tw2, tw3, tid);

        // ---- overlap-add at the delay-compensated positions t = gP - L/2 + n (hop g) and + P (hop g+1), kept to this
        //      CTA's hops.  Slots hit twice (n and n - P) belong to the same thread: no race. ----
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const float2* Y = F + j * kPad;
            float* rj = ring + j * kRing;
            const int base = g * kHop - (p.job[j].L >> 1) - t_lo;
            // length of the linear convolution; the rest of the transform holds only round-off and must not spill into
            // later hops (nor wrap around the ring)
            const int nvalid = kHop + p.job[j].L - 1;
#pragma unroll
            for (int u = 0; u < kN / kThreads; ++u) {
                const int n = tid + u * kThreads;
                const float2 v = Y[padi(n)];
                const int ra = base + n, rb = ra + kHop;
                const bool live = n < nvalid;
                if (live && has_a && ra >= 0 && ra < t_hi - t_lo) rj[ra & (kRing - 1)] += v.y * (1.0f / kN);
                if (live && has_b && rb >= 0 && rb < t_hi - t_lo) rj[rb & (kRing - 1)] += v.x * (1.0f / kN);
            }
        }
        __syncthreads();
        // complete now: every hop below the last input hop just added
        if (g - 1 >= h0 && g - 1 < h1) emit(g - 1);
        if (has_b && g >= h0 && g < h1) emit(g);
        // no barrier needed here: emit touches only the rings, the next iteration's loads only F (whose last reads
        // were ordered by the barrier above), and the rings are next written after the FFT passes' barriers
    }
    if (ge < h1) emit(ge);                        // last hop of the utterance: no following input hop
}

// ---- impulse responses -> packed N-point spectra, once per frame (the SPEC variant of the FIR kernel reads them) ----
// grid (frame groups of 8, utterance, job); frames 2m and 2m+1 of an utterance share one complex transform (pairs never
// cross utterances and do not depend on the batch split: bit-identical output for any sharding); zero upper half -> pruned
// first pass.  Row layout: N/2 float2 per frame, [0] = (H[0], H[N/2]) (both real), [k] = H[k].
struct IrSpecParams {
    const float* ir[2];
    float2* spec[2];
    int L[2];
    int nF;
};

template <int N, bool PK>
__global__ void __launch_bounds__(kThreads) ir_spectrum_kernel(IrSpecParams p) {
    constexpr int kN = N, kPad = Plan<N>::kPad, kTw2 = Plan<N>::kTw2, kTw3 = Plan<N>::kTw3, kQ = 4;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* F = reinterpret_cast<float2*>(smem_raw);
    float2* tw2 = F + kQ * kPad;
    float2* tw3 = tw2 + kTw2;
    const int tid = threadIdx.x, b = blockIdx.y, j = blockIdx.z, nF = p.nF, L = p.L[j];
    const int f0 = blockIdx.x * 2 * kQ;
    const float* ir = p.ir[j] + (size_t)b * nF * L;
    float2* spec = p.spec[j] + (size_t)b * nF * (kN / 2);
    init_twiddles<N>(tw2, tw3, tid);
#pragma unroll
    for (int q = 0; q < kQ; ++q) {
        const int fa = f0 + 2 * q, fb = fa + 1;
        const float* ra = ir + (size_t)min(fa, nF - 1) * L;
        const float* rb = ir + (size_t)min(fb, nF - 1) * L;
        float2* buf = F + q * kPad;
#pragma unroll
        for (int u = 0; u < kN / 2 / kThreads; ++u) {
            const int tau = tid + u * kThreads;
            const bool in = tau < L;
            buf[padi(tau)] = make_float2((in && fa < nF) ? __ldg(ra + tau) : 0.f, (in && fb < nF) ? __ldg(rb + tau) : 0.f);
        }
    }
    __syncthreads();
    fft_forward<N, kQ, PK, true>(F, tw2, tw3, tid);
#pragma unroll
    for (int q = 0; q < kQ; ++q) {
        const int fa = f0 + 2 * q, fb = fa + 1;
        const float2* Z = F + q * kPad;
#pragma unroll
        for (int u = 0; u < kN / 2 / kThreads; ++u) {
            const int k = tid + u * kThreads;
            float2 A, C;
            if (k == 0) {
                const float2 z0 = Z[padi(0)], zN = Z[padi(kN / 2)];
                A = make_float2(z0.x, zN.x);
                C = make_float2(z0.y, zN.y);
            } else {
                split2(Z[padi(k)], Z[padi(kN - k)], A, C);
            }
            if (fa < nF) spec[(size_t)fa * (kN / 2) + k] = A;
            if (fb < nF) spec[(size_t)fb * (kN / 2) + k] = C;
        }
    }
}

}  // namespace

#ifndef B2D_HOST_EMU
namespace b2d {

// block size 512; both jobs' tap counts decide the transform size: <= 512 -> 1024 points, <= 1024 -> 2048 points
bool ltv_fir_fft_supported(int P, int taps1, int taps2, int njobs) {
    const int tmax = njobs == 2 ? (taps1 > taps2 ? taps1 : taps2) : taps1;
    return P == kHop && taps1 > 0 && (njobs == 1 || taps2 > 0) && tmax <= 1024;
}

template <int N, int NJ, bool PK, int NBANK = 0, bool SPEC = false>
static int launch_fir_fft_as(const FftFirParams& p, dim3 grid, cudaStream_t st) {
    constexpr size_t smem = fir_fft_smem<N, NJ, NBANK, SPEC>();
    // per launch, like the direct-form kernels: function attributes are per device and this costs ~1 us
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(ltv_fir_fft_kernel<N, NJ, PK, NBANK, SPEC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return fail((int)e, "ltv_fir(fft): smem attr: %s", cudaGetErrorString(e));
    }
    cudaFuncSetAttribute(ltv_fir_fft_kernel<N, NJ, PK, NBANK, SPEC>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    ltv_fir_fft_kernel<N, NJ, PK, NBANK, SPEC><<<grid, kThreads, smem, st>>>(p);
    return check_launch("ltv_fir(fft)");
}

template <int N, int NJ>
static int launch_fir_fft(const FftFirParams& p, dim3 grid, cudaStream_t st) {
    return g_fft_packed.load(std::memory_order_relaxed) ? launch_fir_fft_as<N, NJ, true>(p, grid, st) : launch_fir_fft_as<N, NJ, false>(p, grid, st);
}

int ltv_fir_fft_launch(const float* x1, const float* ir1, int taps1, float* y1, const float* x2, const float* ir2,
                       int taps2, float* y2, const float* addend, float* mix, uint64_t seed, int64_t utt_off, int B,
                       int nF, int P, cudaStream_t st) {
    const int njobs = ir2 ? 2 : 1;
    if (!ltv_fir_fft_supported(P, taps1, taps2, njobs))
        return fail(B2D_ERR_UNSUPPORTED, "ltv_fir(fft): needs block size %d and at most 1024 taps", kHop);
    FftFirParams p = {};
    p.job[0] = {x1, ir1, y1, taps1};
    p.job[1] = {x2, ir2, y2, njobs == 2 ? taps2 : taps1};
    p.addend = addend; p.mix = mix; p.seed = seed; p.utt_off = utt_off; p.nF = nF;
    // Hops per CTA.  A CTA walks its G + 2 input hops serially (~5.5 us per hop), so G = 32 is right when the grid fills
    // the GPU (B = 32 x 10 s: 864 CTAs for 444 resident slots) but makes small launches -- one utterance of a real-time
    // caller, one chunk of the host pipeline -- latency-bound; halve G (25 % / 50 % / 100 % recomputation at 8 / 4 / 2)
    // until there are at least two CTAs per SM.
    int G = 32;
    while (G > 2 && (long long)B * ((nF + G - 1) / G) < (long long)b2d::num_sms() * 2) G >>= 1;
    p.G = G;
    const dim3 grid((unsigned)((nF + p.G - 1) / p.G), B);
    const int tmax = njobs == 2 ? (taps1 > taps2 ? taps1 : taps2) : taps1;
    if (tmax <= kHop) return njobs == 2 ? launch_fir_fft<1024, 2>(p, grid, st) : launch_fir_fft<1024, 1>(p, grid, st);
    return njobs == 2 ? launch_fir_fft<2048, 2>(p, grid, st) : launch_fir_fft<2048, 1>(p, grid, st);
}

// Sins fused: harmonic = allpass(bank(f0, amplitudes)), noise = filter(white noise), signal = harmonic + noise in ONE
// kernel (block size 512, two filters of at most 512 taps, at most 128 harmonics).
bool sins_fused_supported(int P, int taps_allpass, int taps_noise, int H) {
    return P == kHop && taps_allpass > 0 && taps_noise > 0 && taps_allpass <= kHop && taps_noise <= kHop &&
           !(taps_allpass & 1) && !(taps_noise & 1) && H > 0 && H <= kBankRow;
}

int sins_fused_launch(const float* f0, const double* frame_phase, const float* c_amp, int64_t ctrl_stride, int H,
                      double sampling_rate, int round_fp32, const float* ir_allpass, int taps_allpass, float* harmonic,
                      const float* noise_in, const float* ir_noise, int taps_noise, float* noise_out, float* signal,
                      uint64_t seed, int64_t utt_off, int B, int nF, int P, cudaStream_t st) {
    if (!sins_fused_supported(P, taps_allpass, taps_noise, H))
        return fail(B2D_ERR_UNSUPPORTED, "sins(fused): needs block size %d, <= %d taps, <= %d harmonics", kHop, kHop, kBankRow);
    const float* ptrs[] = {noise_in, harmonic, noise_out, signal};
    for (const float* q : ptrs)
        if (q && !aligned16(q)) return fail(B2D_ERR_ALIGN, "sins(fused): signal pointers must be 16-byte aligned");
    if (B > 65535) return fail(B2D_ERR_UNSUPPORTED, "sins(fused): batch %d > 65535", B);
    FftFirParams p;
    p.job[0] = {nullptr, ir_allpass, harmonic, taps_allpass};
    p.job[1] = {noise_in, ir_noise, noise_out, taps_noise};
    p.addend = nullptr; p.mix = signal; p.seed = seed; p.utt_off = utt_off; p.nF = nF;
    p.bank.f0 = f0; p.bank.frame_phase = frame_phase; p.bank.c_amp = c_amp; p.bank.ctrl_stride = ctrl_stride;
    p.bank.H = H; p.bank.inv_sr = 1.0 / sampling_rate; p.bank.nyquist = (float)(sampling_rate / 2.0);
    p.bank.round_fp32 = round_fp32;
    int G = 32;
    while (G > 2 && (long long)B * ((nF + G - 1) / G) < (long long)b2d::num_sms() * 2) G >>= 1;
    p.G = G;
    const dim3 grid((unsigned)((nF + p.G - 1) / p.G), B);
    const bool pk = g_fft_packed.load(std::memory_order_relaxed) != 0;
    if (H <= 64) return pk ? launch_fir_fft_as<1024, 2, true, 4>(p, grid, st) : launch_fir_fft_as<1024, 2, false, 4>(p, grid, st);
    return pk ? launch_fir_fft_as<1024, 2, true, 8>(p, grid, st) : launch_fir_fft_as<1024, 2, false, 8>(p, grid, st);
}

// ---- spectrum path (Sins): ir_spectrum_kernel once per call, then the SPEC variant of the FIR kernel ----
bool fir_spec_supported(int P, int taps1, int taps2) {
    return P == kHop && taps1 > 0 && taps2 > 0 && taps1 <= kHop && taps2 <= kHop && !(taps1 & 1) && !(taps2 & 1);
}
size_t fir_spec_floats(int B, int nF) { return (size_t)B * nF * 1024; }        // N/2 float2 per frame

int ir_spectrum_launch(const float* ir1, int taps1, float* spec1, const float* ir2, int taps2, float* spec2, int B, int nF,
                       cudaStream_t st) {
    if (!fir_spec_supported(kHop, taps1, taps2)) return fail(B2D_ERR_UNSUPPORTED, "ir_spectrum: needs <= %d taps", kHop);
    if (!aligned16(spec1) || !aligned16(spec2)) return fail(B2D_ERR_ALIGN, "ir_spectrum: spectra must be 16-byte aligned");
    if (B > 65535) return fail(B2D_ERR_UNSUPPORTED, "ir_spectrum: batch %d > 65535", B);
    IrSpecParams p;
    p.ir[0] = ir1; p.ir[1] = ir2; p.L[0] = taps1; p.L[1] = taps2; p.nF = nF;
    p.spec[0] = reinterpret_cast<float2*>(spec1); p.spec[1] = reinterpret_cast<float2*>(spec2);
    constexpr size_t smem = (size_t)4 * Plan<1024>::kPad * sizeof(float2) + (size_t)(Plan<1024>::kTw2 + Plan<1024>::kTw3) * sizeof(float2);
    const dim3 grid((unsigned)((nF + 7) / 8), B, 2);
    if (g_fft_packed.load(std::memory_order_relaxed)) ir_spectrum_kernel<1024, true><<<grid, kThreads, smem, st>>>(p);
    else ir_spectrum_kernel<1024, false><<<grid, kThreads, smem, st>>>(p);
    return check_launch("ir_spectrum");
}

int ltv_fir_fft_spec_launch(const float* x1, const float* spec1, int taps1, float* y1, const float* x2, const float* spec2,
                            int taps2, float* y2, float* mix, uint64_t seed, int64_t utt_off, int B, int nF, int P, cudaStream_t st) {
    if (!fir_spec_supported(P, taps1, taps2)) return fail(B2D_ERR_UNSUPPORTED, "ltv_fir(spec): needs block %d and <= %d taps", kHop, kHop);
    const float* ptrs[] = {x1, x2, y1, y2, mix};
    for (const float* q : ptrs)
        if (q && !aligned16(q)) return fail(B2D_ERR_ALIGN, "ltv_fir(spec): signal pointers must be 16-byte aligned");
    if (B > 65535) return fail(B2D_ERR_UNSUPPORTED, "ltv_fir(spec): batch %d > 65535", B);
    FftFirParams p = {};
    p.job[0] = {x1, spec1, y1, taps1};
    p.job[1] = {x2, spec2, y2, taps2};
    p.addend = nullptr; p.mix = mix; p.seed = seed; p.utt_off = utt_off; p.nF = nF;
    int G = 32;
    while (G > 2 && (long long)B * ((nF + G - 1) / G) < (long long)b2d::num_sms() * 2) G >>= 1;
    p.G = G;
    const dim3 grid((unsigned)((nF + p.G - 1) / p.G), B);
    return g_fft_packed.load(std::memory_order_relaxed) ? launch_fir_fft_as<1024, 2, true, 0, true>(p, grid, st)
                                                        : launch_fir_fft_as<1024, 2, false, 0, true>(p, grid, st);
}

}  // namespace b2d
#endif  // B2D_HOST_EMU
