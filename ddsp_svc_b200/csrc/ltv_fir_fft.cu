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
//     in-place passes below (three block barriers per batch), then all inverse transforms as a second batch;
//   * the two output segments of a pair (P + L - 1 samples each, at their delay-compensated positions) are summed in
//     registers over the pair's output window; its first 2P samples are then complete and written exactly once
//     (y1, y2 and mix = y1 + y2 (+ addend)) with 128-bit stores, the L - 1 samples the next pair also reaches are
//     carried to it -- deterministic, no atomics, no shared-memory ring.
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
static_assert(kHop == 4 * kThreads, "a thread loads and writes 4 samples of every hop");

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
// ---- the kernel's N-point transform: in-place mixed radix (16, N/128, 8) over a batch of padded buffers ----
// Forward = decimation in frequency: natural order in, bin k out at position binpos(k) (digit-reversed).  The transposed
// network (passes in reverse order, twiddles before the butterflies) is again a forward DFT, one that reads that order
// and writes natural order, so the pointwise step runs in place between the two and nothing is ever permuted.  Every
// butterfly writes back the slots it read, so each pass needs ONE block barrier, whatever the batch size (the
// Stockham passes of fft_smem.cuh need one per stage of one or two transforms), and only one butterfly is live per
// thread.  Buffers keep the padding of fft_smem.cuh (slot padi(n)): the slots of a butterfly are the slot of its first
// element plus constants (immediate offsets, no per-element index registers), and with the block order of pass 2 and
// the bin ownership of the pointwise step (own_pos) every half warp hits 16 different bank pairs.
template <int N> struct Ct {
    static_assert(N == 1024 || N == 2048, "supported sizes");
    static constexpr int kM = N / 16;                // span of pass 1
    static constexpr int kR2 = N / 128;              // radix of pass 2 (span 8)
    static constexpr int kTw1 = 8 * kM;              // W_N^(j q) at [(q-1) kM + j], q = 1..8, j < kM (q > 8: times W_N^(8 j))
    static constexpr int kTw2 = 8 * (kR2 - 1);       // W_kM^(j q) at [(q-1) 8 + j], q = 1..kR2-1, j < 8
};
// position of bin k = q + 16 q2 + (N/8) m3 after the forward transform, and its inverse
template <int N> __device__ __forceinline__ int binpos(int k) {
    return (N / 16) * (k & 15) + 8 * ((k >> 4) & (N / 128 - 1)) + k / (N / 8);
}
template <int N> __device__ __forceinline__ int bin_at(int pos) {
    return pos / (N / 16) + 16 * ((pos >> 3) & (N / 128 - 1)) + (N / 8) * (pos & 7);
}
// bins of the pointwise step owned by thread tid: positions 8 (tid + 128 v) + u, u < 4 -- exactly the bins below N/2
// (m3 < 4), consecutive slots across a half warp
__device__ __forceinline__ int own_pos(int tid, int i) { return 8 * (tid + kThreads * (i >> 2)) + (i & 3); }

template <int N> __device__ __forceinline__ void ct_twiddles(float2* tw1, float2* tw2, int tid) {
    constexpr int M = Ct<N>::kM;
    for (int i = tid; i < Ct<N>::kTw1; i += kThreads) {
        const int q = i / M + 1, j = i % M;
        float sn, cs; sincospif(-2.0f * (float)(j * q) / (float)N, &sn, &cs);
        tw1[i] = make_float2(cs, sn);
    }
    for (int i = tid; i < Ct<N>::kTw2; i += kThreads) {
        const int q = i / 8 + 1, j = i % 8;
        float sn, cs; sincospif(-2.0f * (float)(j * q) / (float)M, &sn, &cs);
        tw2[i] = make_float2(cs, sn);
    }
}

// W_N^(j q), q = 1..15, of pass 1 (w = tw1 + j)
template <int N> __device__ __forceinline__ float2 tw_pass1(const float2* w, int q) {
    constexpr int M = Ct<N>::kM;
    return q <= 8 ? w[(q - 1) * M] : cmul(w[(q - 9) * M], w[7 * M]);
}

// pass 1: radix 16 over {j + M r}.  FWD: butterfly, then output q times W_N^(j q); transposed: input r times W_N^(j r),
// then butterfly.  ZU (forward only): the upper half of every transform is zero and is not read.
template <int N, int NB, bool FWD, bool ZU, bool PK>
__device__ __forceinline__ void ct_pass1(float2* F, const float2* tw1, int tid) {
    constexpr int M = Ct<N>::kM, TPJ = kThreads / M, kPad = Plan<N>::kPad;   // TPJ transforms side by side
    const int j = tid % M;
    const float2* w = tw1 + j;
#pragma unroll 1
    for (int u = 0; u < (NB + TPJ - 1) / TPJ; ++u) {
        const int t = tid / M + TPJ * u;
        if (t >= NB) break;
        float2* x = F + t * kPad + padi(j);                     // element r at x[r (M + M/16)]
        float2 v[16];
        if (FWD) {
#pragma unroll
            for (int r = 0; r < (ZU ? 8 : 16); ++r) v[r] = x[r * (M + M / 16)];
            if (ZU) Dft16ZeroUpper<PK>::run(v);
            else Dft<16, PK>::run(v);
#pragma unroll
            for (int q = 1; q < 16; ++q) v[q] = cmul(v[q], tw_pass1<N>(w, q));
        } else {
            v[0] = x[0];
#pragma unroll
            for (int r = 1; r < 16; ++r) v[r] = cmul(x[r * (M + M / 16)], tw_pass1<N>(w, r));
            Dft<16, PK>::run(v);
        }
#pragma unroll
        for (int q = 0; q < 16; ++q) x[q * (M + M / 16)] = v[q];
    }
}

// pass 2: radix R2 over {M q + j + 8 r} inside each of the 16 blocks of pass 1, twiddles W_M^(j r).  For N = 1024 the
// two 8-lane groups of a half warp take blocks two apart (bits 0 and 1 of the block index swapped): their slots are
// then 8 banks pairs apart, as they are for neighbouring blocks when N = 2048.
template <int N, int NB, bool FWD, bool PK>
__device__ __forceinline__ void ct_pass2(float2* F, const float2* tw2, int tid) {
    constexpr int M = Ct<N>::kM, R2 = Ct<N>::kR2, kPad = Plan<N>::kPad;
    const int j = tid & 7, b = tid >> 3;
    const int q = N == 1024 ? ((b & ~3) | ((b & 1) << 1) | ((b >> 1) & 1)) : b;
    const float2* w = tw2 + j;
#pragma unroll 1
    for (int t = 0; t < NB; ++t) {
        float2* x = F + t * kPad + padi(M * q + j);            // element r at x[8 r + r / 2]
        float2 v[R2];
        v[0] = x[0];
#pragma unroll
        for (int r = 1; r < R2; ++r) {
            v[r] = x[8 * r + r / 2];
            if (!FWD) v[r] = cmul(v[r], w[(r - 1) * 8]);
        }
        Dft<R2, PK>::run(v);
        if (FWD) {
#pragma unroll
            for (int r = 1; r < R2; ++r) v[r] = cmul(v[r], w[(r - 1) * 8]);
        }
#pragma unroll
        for (int r = 0; r < R2; ++r) x[8 * r + r / 2] = v[r];
    }
}

// pass 3: radix 8 over 8 consecutive positions, no twiddles (its own transpose)
template <int N, int NB, bool PK>
__device__ __forceinline__ void ct_pass3(float2* F, int tid) {
    constexpr int kPad = Plan<N>::kPad;
#pragma unroll 1
    for (int i = tid; i < NB * (N / 8); i += kThreads) {
        float2* x = F + (i / (N / 8)) * kPad + padi(8 * (i % (N / 8)));
        float2 v[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) v[r] = x[r];
        Dft<8, PK>::run(v);
#pragma unroll
        for (int r = 0; r < 8; ++r) x[r] = v[r];
    }
}

// NB transforms at F, F + kPad, ...: natural order -> bin k at position binpos(k) (ct_forward) and back
// (ct_transposed); both end with a barrier
template <int N, int NB, bool PK, bool ZU = false>
__device__ __forceinline__ void ct_forward(float2* F, const float2* tw1, const float2* tw2, int tid) {
    ct_pass1<N, NB, true, ZU, PK>(F, tw1, tid);
    __syncthreads();
    ct_pass2<N, NB, true, PK>(F, tw2, tid);
    __syncthreads();
    ct_pass3<N, NB, PK>(F, tid);
    __syncthreads();
}
// (`after_pass3` runs between the first pass and its barrier)
template <int N, int NB, bool PK, class AfterPass3>
__device__ __forceinline__ void ct_transposed(float2* F, const float2* tw1, const float2* tw2, int tid, AfterPass3 after_pass3) {
    ct_pass3<N, NB, PK>(F, tid);
    after_pass3();
    __syncthreads();
    ct_pass2<N, NB, false, PK>(F, tw2, tid);
    __syncthreads();
    ct_pass1<N, NB, false, false, PK>(F, tw1, tid);
    __syncthreads();
}

// SPEC variant: the spectra of the impulse responses are read from memory (ir_spectrum_kernel made them once per frame),
// so the HH buffers and a quarter of the transforms disappear: 2 NJ buffers -> 54.4 KB for N = 1024, NJ = 2 -> 4 CTAs per SM
template <int N, int NJ, int NBANK = 0, bool SPEC = false> constexpr size_t fir_fft_smem() {
    return (size_t)(SPEC ? 2 : 3) * NJ * Plan<N>::kPad * sizeof(float2) + (size_t)(Ct<N>::kTw1 + Ct<N>::kTw2) * sizeof(float2) +
           (NBANK ? (size_t)5 * kBankRow * sizeof(float) : 0);
}   // N = 1024: NJ = 2 -> 56768 B (4 CTAs per SM), NJ = 1 -> 30656 B;  N = 2048: NJ = 1 -> 61376 B, NJ = 2 -> 113600 B
// __launch_bounds__ minimum: the two-job 1024-point kernels (taps or spectra) fit 4 CTAs per SM in shared memory
// (4 x (56768 + 1024 reserved) B <= 228 KB) and hold <= 128 registers without spilling; the bank variant needs more.
template <int N, int NJ, int NBANK> constexpr int fir_fft_min_ctas() {
    return (N == 2048 && NJ == 2) ? 1 : (N == 1024 && NJ == 2 && NBANK == 0) ? 4 : 3;
}

// spectra of two real sequences a, c from Z = FFT(a + j c):  A[k] = (Z[k] + conj Z[N-k]) / 2,  C[k] = (Z[k] - conj Z[N-k]) / 2j
__device__ __forceinline__ void split2(float2 zk, float2 zm, float2& A, float2& C) {
    A = make_float2(0.5f * (zk.x + zm.x), 0.5f * (zk.y - zm.y));
    C = make_float2(0.5f * (zk.y + zm.y), 0.5f * (zm.x - zk.x));
}

// PK: the "packed" complex-addition policy (fft_regs.cuh Ar<true>; scalar on Hopper)
// NBANK: 0 = inputs from memory / Philox; 4 or 8 = job 0 is the sinusoid bank with that many bases of 16 harmonics
// SPEC: job[j].ir holds the packed 1024-point spectra of the impulse responses instead of the taps
template <int N, int NJ, bool PK, int NBANK = 0, bool SPEC = false>
__global__ void __launch_bounds__(kThreads, fir_fft_min_ctas<N, NJ, NBANK>()) ltv_fir_fft_kernel(FftFirParams p) {
    constexpr int kN = N, kPad = Plan<N>::kPad;
    constexpr int kBins = N / 2 / kThreads;          // bins per thread (own_pos: DC .. N/2-1); Nyquist on thread 0
    extern __shared__ __align__(16) unsigned char smem_raw[];
    // buffer b of the batch lives at F + b * kPad:  XA(j) = j  (hop g; later the paired output of job j),
    // XB(j) = NJ + j (hop g+1),  HH(j) = 2 NJ + j (impulse responses of frames g+1 and g+2).  Sample n of a buffer is at
    // slot padi(n), bin k of a forward-transformed one at slot at(k).
    float2* F = reinterpret_cast<float2*>(smem_raw);
    float2* tw1 = F + (SPEC ? 2 : 3) * NJ * kPad;
    float2* tw2 = tw1 + Ct<N>::kTw1;
    float* bank_act = reinterpret_cast<float*>(tw2 + Ct<N>::kTw2);   // BANK: [3][128] activated amplitudes of frames g, g+1, g+2
    float* bank_dlt = bank_act + 3 * kBankRow;                   //       [2][128] their differences

    const int tid = threadIdx.x;
    const int b = blockIdx.y;
    const int nF = p.nF, T = nF * kHop;
    const int h0 = blockIdx.x * p.G, h1 = min(h0 + p.G, nF);
    const int t_lo = h0 * kHop, t_hi = h1 * kHop;
    const unsigned long long utt = (unsigned long long)(p.utt_off + b);

    ct_twiddles<N>(tw1, tw2, tid);
    auto at = [](int k) { return padi(binpos<N>(k)); };
    const auto own_bin = [&](int u) { return bin_at<N>(own_pos(tid, u)); };

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
    // They land in shared memory as soon as the previous pair has freed it (stage), so the registers are not held
    // through that pair's inverse transforms and overlap-add.
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
    // Taps go to the HH buffers.  Input samples go unchanged to the upper half of XB(j), which the transforms do not read
    // (zero upper halves) and load_x does not write; each thread reads back only its own samples.
    auto xstage = [&](int j, int hop) { return F + (NJ + j) * kPad + padi(kN / 2 + hop * (kHop / 2) + (tid << 1)); };
    auto stage = [&](const Prefetch& q) {
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            if (!SPEC) {
                float2* buf = F + (2 * NJ + j) * kPad;
#pragma unroll
                for (int u = 0; u < kTau; ++u) buf[padi(tid + u * kThreads)] = make_float2(q.ha[j][u], q.hb[j][u]);
            }
            if (p.job[j].x && !(NBANK && j == 0)) {
                xstage(j, 0)[0] = make_float2(q.xa[j].x, q.xa[j].y);
                xstage(j, 0)[1] = make_float2(q.xa[j].z, q.xa[j].w);
                xstage(j, 1)[0] = make_float2(q.xb[j].x, q.xb[j].y);
                xstage(j, 1)[1] = make_float2(q.xb[j].z, q.xb[j].w);
            }
        }
    };
    auto staged_x = [&](int j, int hop) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p.job[j].x) {
            const float2 lo = xstage(j, hop)[0], hi = xstage(j, hop)[1];
            v = make_float4(lo.x, lo.y, hi.x, hi.y);
        }
        return v;
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

    // spectrum of frame g per job at the bins own_bin(u); thread 0 holds the real DC and Nyquist values as (DC, Nyquist) at u = 0
    float2 Hp[NJ][kBins];
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
                const int k = own_bin(u);
                Hp[j][u] = __ldg(row + k);                              // row[0] = (DC, Nyquist) as well
            }
        }
        __syncthreads();                                                // twiddles
    } else {
#pragma unroll
        for (int j = 0; j < NJ; ++j) load_ir_pair(j, gs - 1, gs, true);    // exactly the (h_{g+1}, h_{g+2}) pair of hops gs-2, gs-1
        __syncthreads();
        ct_forward<N, NJ, PK, true>(F + 2 * NJ * kPad, tw1, tw2, tid);
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            const float2* H = F + (2 * NJ + j) * kPad;
#pragma unroll
            for (int u = 0; u < kBins; ++u) {
                const int k = own_bin(u);
                float2 unused;
                if (k == 0) Hp[j][u] = make_float2(H[at(0)].y, H[at(kN / 2)].y);
                else split2(H[padi(own_pos(tid, u))], H[at(kN - k)], unused, Hp[j][u]);
            }
        }
        __syncthreads();
    }

    // Output window of the pair that starts at input hop g: samples t = gP - A + w, w < 2P + N/2, where thread tid owns
    // w = P c + 4 tid + e (e < 4).  A, the larger half tap count rounded up to 4, puts every job's segments at or after
    // the window's start and keeps the 128-bit stores aligned.  Samples w < 2P are final after the pair: the next pair's
    // segments start at (g+2)P - L/2 >= (g+2)P - A.  The rest, at most L - 1 samples per job, is the head of the next
    // window, where the same thread owns it, so it is carried in registers.
    constexpr int kCarry = N / 2 / kHop;              // hop-long chunks of a window carried into the next one
    int A = p.job[0].L >> 1;
    if (NJ == 2) A = max(A, p.job[1].L >> 1);
    A = (A + 3) & ~3;
    float carry[NJ][kCarry][4];
#pragma unroll
    for (int j = 0; j < NJ; ++j)
#pragma unroll
        for (int c = 0; c < kCarry; ++c)
#pragma unroll
            for (int e = 0; e < 4; ++e) carry[j][c][e] = 0.f;

    // write the 4 samples from t (a multiple of 4) of y_j and mix, if they belong to this CTA's hops
    auto emit = [&](int t, const float4 (&v)[NJ]) {
        if (t < t_lo || t >= t_hi) return;
        const size_t o = (size_t)b * T + t;
        float4 m = v[0];
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
            if (p.job[j].y) b2d::st_global_v4(p.job[j].y + o, v[j]);
            if (j > 0) { m.x += v[j].x; m.y += v[j].y; m.z += v[j].z; m.w += v[j].w; }
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
    stage(pf);
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
                const float4 xa = staged_x(j, 0), xb = staged_x(j, 1);
                load_x(j, g, has_a, xa, F + j * kPad);
                load_x(j, g + 1, has_b, xb, F + (NJ + j) * kPad);
            }
        }
        __syncthreads();
        ct_forward<N, (SPEC ? 2 : 3) * NJ, PK, true>(F, tw1, tw2, tid);   // all have zero upper halves: pruned first pass

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
                for (int u = 0; u < kBins; ++u) { HaR[u] = __ldg(rowA + own_bin(u)); HbR[u] = __ldg(rowB + own_bin(u)); }
            }
#pragma unroll
            for (int u = 0; u < kBins; ++u) {
                const int k = own_bin(u);
                if (k == 0) continue;
                const int ik = padi(own_pos(tid, u)), im = at(kN - k);
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
                const float2 a0 = XA[at(0)], b0 = XB[at(0)];                              // (X, XU), (X, XU)
                const float2 aN = XA[at(kN / 2)], bN = XB[at(kN / 2)];
                // (H_{g+1}, H_{g+2}) at DC and at Nyquist
                const float2 z0 = SPEC ? make_float2(HaR[0].x, HbR[0].x) : HH[at(0)];
                const float2 zN = SPEC ? make_float2(HaR[0].y, HbR[0].y) : HH[at(kN / 2)];
                const float hp0 = Hp[j][0].x, hpN = Hp[j][0].y;
                const float ya0 = fmaf(a0.y, z0.x - hp0, a0.x * hp0), yb0 = fmaf(b0.y, z0.y - z0.x, b0.x * z0.x);
                const float yaN = fmaf(aN.y, zN.x - hpN, aN.x * hpN), ybN = fmaf(bN.y, zN.y - zN.x, bN.x * zN.x);
                XA[at(0)] = make_float2(yb0, ya0);
                XA[at(kN / 2)] = make_float2(ybN, yaN);
                Hp[j][0] = make_float2(z0.y, zN.y);
            }
        }
        __syncthreads();
        // the next pair's loads fly during the first inverse pass (issued here, not earlier: the registers they land
        // in would otherwise be held through the forward batch and the pointwise step)
        if (g + 2 <= ge) fetch(g + 2, pf);

        // ---- inverse of the pairs (batch over jobs): hop g = stored .y / N, hop g+1 = stored .x / N.  The next pair's
        //      loads are staged after the first pass: XB and HH are free since the pointwise step. ----
        ct_transposed<N, NJ, PK>(F, tw1, tw2, tid, [&] { if (g + 2 <= ge) stage(pf); });

        // ---- overlap-add over the pair's output window: job j's segments of hops g and g+1 start at w = d and d + P
        //      (d = A - L/2); carried head + hop g+1 + hop g, the order in which a running sum would meet them.  The
        //      final part is written, the tail carried. ----
#pragma unroll
        for (int c = 0; c < 2 + kCarry; ++c) {
            float4 v[NJ];
#pragma unroll
            for (int j = 0; j < NJ; ++j) {
                const float2* Y = F + j * kPad;
                // length of the linear convolution; the rest of the transform holds only round-off and must not reach
                // later samples
                const int nvalid = kHop + p.job[j].L - 1;
                const int n0 = kHop * c + (tid << 2) - (A - (p.job[j].L >> 1));
                float s[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int na = n0 + e, nb = na - kHop;
                    float acc = c < kCarry ? carry[j][c < kCarry ? c : 0][e] : 0.f;
                    // hop g+1 reaches w >= P, hop g only w < P + N/2 (L <= N/2, A <= N/4)
                    if (c >= 1 && has_b && nb >= 0 && nb < nvalid) acc += Y[padi(nb)].x * (1.0f / kN);
                    if (c <= kCarry && has_a && na >= 0 && na < nvalid) acc += Y[padi(na)].y * (1.0f / kN);
                    s[e] = acc;
                }
                v[j] = make_float4(s[0], s[1], s[2], s[3]);
                if (c >= 2) {
#pragma unroll
                    for (int e = 0; e < 4; ++e) carry[j][c >= 2 ? c - 2 : 0][e] = s[e];
                }
            }
            if (c < 2) emit(g * kHop - A + kHop * c + (tid << 2), v);
        }
        // the next iteration's loads overwrite the Y buffers read above
        __syncthreads();
    }
    // the carried tail of the last window: output only where no later input hop reaches (the end of the utterance)
    const int g_end = gs + 2 * ((ge - gs) / 2 + 1);
#pragma unroll
    for (int c = 0; c < kCarry; ++c) {
        float4 v[NJ];
#pragma unroll
        for (int j = 0; j < NJ; ++j) v[j] = make_float4(carry[j][c][0], carry[j][c][1], carry[j][c][2], carry[j][c][3]);
        emit(g_end * kHop - A + kHop * c + (tid << 2), v);
    }
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

// Hops per CTA, G (even).  A CTA walks its G + 2 input hops serially, so a launch takes about
// (waves of CTAs at the kernel's occupancy) x (G + 2) hop times.  On B = 32 x 10 s (nF = 861) at 4 CTAs per SM (528
// slots on 132 SMs) that is G = 54: 512 CTAs in one wave, 56 hop times (at 3 CTAs per SM: G = 36, 768 CTAs in two
// waves of 396, 76 hop times).  Pick the G that minimises that product (the largest on a tie:
// least recomputation); it also shrinks G for small launches -- one utterance of a real-time caller, one chunk of the
// host pipeline -- until they spread over the GPU.  The output does not depend on G (hops are always paired the same way).
// `occ` caches the occupancy per device: the query costs host time that a small (real-time) launch would notice.
static int fir_fft_hops_per_cta(const void* kernel, size_t smem, std::atomic<int>* occ, int B, int nF) {
    constexpr int kMaxHops = 64;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) { cudaGetLastError(); dev = -1; }
    int per_sm = dev >= 0 ? occ[dev].load(std::memory_order_relaxed) : 0;
    if (per_sm <= 0) {
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, smem) != cudaSuccess || per_sm < 1) {
            cudaGetLastError();
            per_sm = 1;
        }
        if (dev >= 0) occ[dev].store(per_sm, std::memory_order_relaxed);
    }
    const long long slots = (long long)per_sm * b2d::num_sms();
    int best = 2;
    long long best_cost = -1;
    for (int G = kMaxHops; G >= 2; G -= 2) {
        const long long ctas = (long long)B * ((nF + G - 1) / G);
        const long long cost = (ctas + slots - 1) / slots * (G + 2);
        if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = G; }
    }
    return best;
}

template <int N, int NJ, bool PK, int NBANK = 0, bool SPEC = false>
static int launch_fir_fft_as(FftFirParams p, int B, cudaStream_t st) {
    const auto kernel = ltv_fir_fft_kernel<N, NJ, PK, NBANK, SPEC>;
    constexpr size_t smem = fir_fft_smem<N, NJ, NBANK, SPEC>();
    // per launch, like the direct-form kernels: function attributes are per device and this costs ~1 us
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return fail((int)e, "ltv_fir(fft): smem attr: %s", cudaGetErrorString(e));
    }
    cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    static std::atomic<int> occ[64];
    p.G = fir_fft_hops_per_cta(reinterpret_cast<const void*>(kernel), smem, occ, B, p.nF);
    const dim3 grid((unsigned)((p.nF + p.G - 1) / p.G), B);
    kernel<<<grid, kThreads, smem, st>>>(p);
    return check_launch("ltv_fir(fft)");
}

template <int N, int NJ>
static int launch_fir_fft(const FftFirParams& p, int B, cudaStream_t st) {
    return g_fft_packed.load(std::memory_order_relaxed) ? launch_fir_fft_as<N, NJ, true>(p, B, st) : launch_fir_fft_as<N, NJ, false>(p, B, st);
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
    const int tmax = njobs == 2 ? (taps1 > taps2 ? taps1 : taps2) : taps1;
    if (tmax <= kHop) return njobs == 2 ? launch_fir_fft<1024, 2>(p, B, st) : launch_fir_fft<1024, 1>(p, B, st);
    return njobs == 2 ? launch_fir_fft<2048, 2>(p, B, st) : launch_fir_fft<2048, 1>(p, B, st);
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
    const bool pk = g_fft_packed.load(std::memory_order_relaxed) != 0;
    if (H <= 64) return pk ? launch_fir_fft_as<1024, 2, true, 4>(p, B, st) : launch_fir_fft_as<1024, 2, false, 4>(p, B, st);
    return pk ? launch_fir_fft_as<1024, 2, true, 8>(p, B, st) : launch_fir_fft_as<1024, 2, false, 8>(p, B, st);
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
    return g_fft_packed.load(std::memory_order_relaxed) ? launch_fir_fft_as<1024, 2, true, 0, true>(p, B, st)
                                                        : launch_fir_fft_as<1024, 2, false, 0, true>(p, B, st);
}

}  // namespace b2d
#endif  // B2D_HOST_EMU
