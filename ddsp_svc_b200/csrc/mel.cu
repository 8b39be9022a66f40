// K8: log-mel spectrogram front end of the NSF-HiFiGAN vocoder -- replaces STFT.get_mel (nsf_hifigan/nvSTFT.py:73-117),
// the consumer of the synthesizer's waveform in enhancer.py:113, diffusion/vocoder.py:147 and reflow/vocoder.py:125:
//
//   y_pad  = pad(y, (win - hop) / 2 each side, reflect | constant)                     (:97-104)
//   S      = stft(y_pad, n_fft = win = 2048, hop, hann (periodic), center = False)       (:106-107)
//   mag    = sqrt(Re^2 + Im^2 + 1e-9)                                                    (:108)
//   mel    = log(clamp(mel_basis [n_mels, 1025] @ mag, clip_val))                        (:114-115)
//
// for the shape every shipped configuration uses (keyshift 0, speed 1: n_fft = win = 2048; any hop, n_mels <= 128).
// One CTA (128 threads) owns 16 consecutive frames of one utterance and transforms them TWO at a time: a complex
// 2048-point FFT of w (ya + j yb) in shared memory (fft_smem.cuh, radix 16 x 16 x 8) carries both real frames, the two
// spectra are separated by conjugate symmetry, and thread m reduces its mel filter over the bins where it is non-zero
// (the triangular filters are sparse: ~2 050 of 131 200 weights; [lo, hi) per filter comes from the host) for both
// frames.  The 128 x 16 results are staged in shared memory and written as 64-byte row segments of the
// [B, n_mels, n_frames] output.  HBM: the waveform is read once (the 4x frame overlap is served by L1/L2), 4 n_mels /
// hop bytes per input sample are written: 4 + 1 = 5 B per sample for 128 mels at hop 512.
//
// mel_bwd_kernel: gradient of the above with respect to y (training: the DDSP loss of the reflow / diffusion models).
// See the comment above the kernel; it shares the framing, FFT, magnitude and projection with mel_kernel, so the mel
// value it recomputes is bit-identical to the forward's and it takes the forward's clamp decision.
#ifndef B2D_HOST_EMU               // tests/emu/ runs the kernels' source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif
#include "bluestein.cuh"

using namespace b2d_fft;
using namespace b2d_bluestein;
using b2d_fft_smem::kThreads;
using b2d_fft_smem::padi;

extern "C" int b2d_mel_frames(int n_samples, int n_fft, int win_size, int hop);

namespace {

constexpr int kN = 2048, kBins = kN / 2 + 1;
constexpr int kPad = b2d_fft_smem::Plan<kN>::kPad, kTw2 = b2d_fft_smem::Plan<kN>::kTw2, kTw3 = b2d_fft_smem::Plan<kN>::kTw3;
constexpr int kFramesPerCta = 16;
constexpr int kMagStride = kBins + 3;                       // 1028 floats per frame of magnitudes
constexpr size_t kSmemBytes = (size_t)kPad * sizeof(float2) + (size_t)(kTw2 + kTw3) * sizeof(float2) +
                              (size_t)2 * kMagStride * sizeof(float) + (size_t)128 * (kFramesPerCta + 1) * sizeof(float);

struct MelParams {
    const float* y;            // [B, T]
    const float* window;       // [2048] hann, periodic (torch.hann_window)
    const float* basis;        // [n_mels, 1025]
    const int* lohi;           // [n_mels, 2] first / one-past-last non-zero bin of each filter
    float* out;                // [B, n_mels, n_frames]
    int T, hop, n_frames, n_mels, pad_left, reflect;
    float clip;
};

__device__ __forceinline__ float sample_at(const float* __restrict__ y, int T, int src, int reflect_mode) {
    if (src >= 0 && src < T) return __ldg(y + src);
    if (!reflect_mode) return 0.f;
    const int r = src < 0 ? -src : 2 * (T - 1) - src;       // torch 'reflect' (pad < T is guaranteed by the host check)
    return __ldg(y + r);
}

// ---- the steps mel_kernel and mel_bwd_kernel share (the backward must recompute the forward's values bit for bit) ----

// windowed frames fa (real part) and fa + 1 (imaginary part; zero when !has_b) of utterance row y into F
__device__ __forceinline__ void load_frame_pair(float2* F, const float* __restrict__ y, const float* __restrict__ window,
                                                int T, int hop, int pad_left, int reflect, int fa, bool has_b, int tid) {
    const int s0 = fa * hop - pad_left;
    if (s0 >= 0 && s0 + hop + kN <= T && has_b) {
        // interior pair (all but the first / last frames): no bounds logic, all 48 loads of a thread in flight at once
        float va[kN / kThreads], vb[kN / kThreads], w[kN / kThreads];
#pragma unroll
        for (int u = 0; u < kN / kThreads; ++u) {
            const int n = tid + u * kThreads;
            w[u] = __ldg(window + n);
            va[u] = __ldg(y + s0 + n);
            vb[u] = __ldg(y + s0 + hop + n);
        }
#pragma unroll
        for (int u = 0; u < kN / kThreads; ++u) F[padi(tid + u * kThreads)] = make_float2(w[u] * va[u], w[u] * vb[u]);
    } else {
#pragma unroll 4
        for (int u = 0; u < kN / kThreads; ++u) {
            const int n = tid + u * kThreads;
            const float w = __ldg(window + n);
            const float va = sample_at(y, T, s0 + n, reflect);
            const float vb = has_b ? sample_at(y, T, s0 + n + hop, reflect) : 0.f;
            F[padi(n)] = make_float2(w * va, w * vb);
        }
    }
}

// A[k], B[k] (k <= 1024) from Z = FFT(a + j b):  A = (Z[k] + conj Z[N-k]) / 2,  B = (Z[k] - conj Z[N-k]) / 2j
__device__ __forceinline__ void split_pair(const float2* F, int k, float& ar, float& ai, float& br, float& bi) {
    const float2 zk = F[padi(k)], zm = F[padi((kN - k) & (kN - 1))];
    ar = 0.5f * (zk.x + zm.x); ai = 0.5f * (zk.y - zm.y);
    br = 0.5f * (zk.y + zm.y); bi = 0.5f * (zm.x - zk.x);
}

// |A[k]|, |B[k]| of the transformed pair in F -> mag[k], mag[kMagStride + k]
__device__ __forceinline__ void pair_magnitudes(const float2* F, float* mag, int tid) {
    for (int k = tid; k < kBins; k += kThreads) {
        float ar, ai, br, bi;
        split_pair(F, k, ar, ai, br, bi);
        mag[k] = sqrtf(ar * ar + ai * ai + 1e-9f);
        mag[kMagStride + k] = sqrtf(br * br + bi * bi + 1e-9f);
    }
}

// mel filter row brow over its support [lo, hi), both frames: the pre-log values M_a, M_b
__device__ __forceinline__ void project_pair(const float* mag, const float* __restrict__ brow, int lo, int hi,
                                             float& sa, float& sb) {
    sa = 0.f; sb = 0.f;
    for (int k = lo; k < hi; ++k) {
        const float wgt = __ldg(brow + k);
        sa = fmaf(wgt, mag[k], sa);
        sb = fmaf(wgt, mag[kMagStride + k], sb);
    }
}

__global__ void __launch_bounds__(kThreads, 3) mel_kernel(MelParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* F = reinterpret_cast<float2*>(smem_raw);
    float2* tw2 = F + kPad;
    float2* tw3 = tw2 + kTw2;
    float* mag = reinterpret_cast<float*>(tw3 + kTw3);        // [2][kMagStride]
    float* stage = mag + 2 * kMagStride;                      // [128][kFramesPerCta + 1]
    const int tid = threadIdx.x, b = blockIdx.y;
    const int f0 = blockIdx.x * kFramesPerCta, f1 = min(f0 + kFramesPerCta, p.n_frames);
    const float* y = p.y + (size_t)b * p.T;

    b2d_fft_smem::init_twiddles<kN>(tw2, tw3, tid);
    int lo = 0, hi = 0;
    if (tid < p.n_mels) { lo = p.lohi[2 * tid]; hi = p.lohi[2 * tid + 1]; }
    const float* brow = p.basis + (size_t)min(tid, p.n_mels - 1) * kBins;

    for (int fa = f0; fa < f1; fa += 2) {
        const bool has_b = fa + 1 < f1;
        // ---- windowed frames fa (real part) and fa + 1 (imaginary part) ----
        load_frame_pair(F, y, p.window, p.T, p.hop, p.pad_left, p.reflect, fa, has_b, tid);
        __syncthreads();
        b2d_fft_smem::fft_forward<kN, 1, true>(F, tw2, tw3, tid);
        // ---- |A[k]|, |B[k]| ----
        pair_magnitudes(F, mag, tid);
        __syncthreads();
        // ---- mel projection: thread m over the support of its filter, both frames ----
        if (tid < p.n_mels) {
            float sa, sb;
            project_pair(mag, brow, lo, hi, sa, sb);
            stage[tid * (kFramesPerCta + 1) + (fa - f0)] = logf(fmaxf(sa, p.clip));
            stage[tid * (kFramesPerCta + 1) + (fa - f0) + 1] = logf(fmaxf(sb, p.clip));
        }
        // the next iteration's loads write F only; mag is rewritten after two more barriers: no barrier needed here
    }
    __syncthreads();
    // ---- write out: row segments of up to 16 frames ----
    const int nfr = f1 - f0;
    for (int i = tid; i < p.n_mels * kFramesPerCta; i += kThreads) {
        const int m = i / kFramesPerCta, c = i - m * kFramesPerCta;
        if (c < nfr) p.out[((size_t)b * p.n_mels + m) * p.n_frames + f0 + c] = stage[m * (kFramesPerCta + 1) + c];
    }
}

// ---- keyshift: STFT.get_mel(y, keyshift) for keyshift != 0 (nvSTFT.py:73-117, speed 1, center False) ----
// n' = round(2048 * 2^(keyshift / 12)) is both the transform and the window length, any integer in [hop, 3072]:
//   y_pad  = pad(y, (n' - hop) / 2 left, max((n' - hop + 1) / 2, n' - T - left) right, reflect | constant)
//   X      = n'-point DFT of hann(n') frames, bins k < K = min(1025, n' / 2 + 1)
//   mag    = sqrt(Re^2 + Im^2 + 1e-9) * 2048 / n' for k < K, exactly 0 for K <= k < 1025 (the pad follows the sqrt)
//   mel    = log(clamp(mel_basis [n_mels, 1025] @ mag, clip_val))   (the unshifted 2048-point basis)
// The DFT is Bluestein's (bluestein.cuh) for the K bins only, so M >= n' + K - 1: 4096 up to n' = 3072.  One CTA owns
// two consecutive frames of one utterance, transformed side by side in one batched FFT.  They are not packed as a + j b
// like mel_kernel's pairs: separating the two spectra needs bins n' - k beyond K, which an M-point convolution this
// small does not produce.  A CTA owns one pair and no loop over pairs: the 4096-point transforms need nearly all 255
// registers, and a frame loop lets the compiler hoist their index arithmetic out of it and spill.
// The table (bluestein.cuh's layout, window hann(n')) is per n'.  The projection is mel_kernel's.
struct MelKeyshiftParams {
    const float* y;            // [B, T]
    const float* table;        // bluestein.cuh table of n (window, chirp, FFT_M(h) / M)
    const float* basis;        // [n_mels, 1025]
    const int* lohi;           // [n_mels, 2]
    float* out;                // [B, n_mels, n_frames]
    int T, hop, n, K, n_frames, n_mels, pad_left, reflect;
    float clip;
};

constexpr int kKeyshiftMaxN = 3072;

template <int M> constexpr size_t keyshift_smem_bytes() {
    return (size_t)2 * b2d_fft_smem::Plan<M>::kPad * sizeof(float2) +
           (size_t)(b2d_fft_smem::Plan<M>::kTw2 + b2d_fft_smem::Plan<M>::kTw3) * sizeof(float2) +
           (size_t)2 * kMagStride * sizeof(float);
}

// ZU: n <= M / 2, the first FFT skips the zero upper half of its input
template <int M, bool ZU>
__global__ void __launch_bounds__(kThreads) mel_keyshift_kernel(MelKeyshiftParams p) {
    constexpr int kPadM = b2d_fft_smem::Plan<M>::kPad;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* z = reinterpret_cast<float2*>(smem_raw);          // [2][kPadM] frames fa, fa + 1
    float2* tw2 = z + 2 * kPadM;
    float2* tw3 = tw2 + b2d_fft_smem::Plan<M>::kTw2;
    float* mag = reinterpret_cast<float*>(tw3 + b2d_fft_smem::Plan<M>::kTw3);        // [2][kMagStride]
    const int tid = threadIdx.x, b = blockIdx.y, n = p.n, fa = 2 * blockIdx.x;
    const bool has_b = fa + 1 < p.n_frames;
    const float* y = p.y + (size_t)b * p.T;
    const float* window = p.table + kWinOff;
    const float2* chirp = reinterpret_cast<const float2*>(p.table + chirp_off(n));

    b2d_fft_smem::init_twiddles<M>(tw2, tw3, tid);
    // ---- windowed, chirped frames fa and fa + 1: w y conj(c) on [0, n), zero above ----
    const int s0 = fa * p.hop - p.pad_left;
    for (int m = tid; m < (ZU ? M / 2 : M); m += kThreads) {
        float2 va = make_float2(0.f, 0.f), vb = va;
        if (m < n) {
            const float w = __ldg(window + m);
            const float2 ch = __ldg(chirp + m);
            const float a = w * sample_at(y, p.T, s0 + m, p.reflect);
            const float c = has_b ? w * sample_at(y, p.T, s0 + p.hop + m, p.reflect) : 0.f;
            va = make_float2(a * ch.x, -a * ch.y);
            vb = make_float2(c * ch.x, -c * ch.y);
        }
        z[padi(m)] = va;
        z[kPadM + padi(m)] = vb;
    }
    __syncthreads();
    bluestein_core<M, 2, ZU>(z, reinterpret_cast<const float2*>(p.table + hspec_off(n)), tw2, tw3, tid);
    // ---- magnitudes of bins k < K, scaled by 2048 / n; zero above ----
    for (int k = tid; k < kBins; k += kThreads) {
        float ma = 0.f, mb = 0.f;
        if (k < p.K) {
            const float2 xa = bluestein_out<M>(z, chirp, k), xb = bluestein_out<M>(z + kPadM, chirp, k);
            ma = sqrtf(xa.x * xa.x + xa.y * xa.y + 1e-9f) * 2048.f / (float)n;
            mb = sqrtf(xb.x * xb.x + xb.y * xb.y + 1e-9f) * 2048.f / (float)n;
        }
        mag[k] = ma;
        mag[kMagStride + k] = mb;
    }
    __syncthreads();
    // ---- mel projection and log: thread m, both frames ----
    if (tid < p.n_mels) {
        float sa, sb;
        project_pair(mag, p.basis + (size_t)tid * kBins, __ldg(p.lohi + 2 * tid), __ldg(p.lohi + 2 * tid + 1), sa, sb);
        float* row = p.out + ((size_t)b * p.n_mels + tid) * p.n_frames + fa;
        row[0] = logf(fmaxf(sa, p.clip));
        if (has_b) row[1] = logf(fmaxf(sb, p.clip));
    }
}

// the shape fields of p for n_samples, n' = n_fft, hop (nvSTFT.py:97-104); returns n_frames (0: no frame)
int keyshift_setup(MelKeyshiftParams& p, int n_samples, int n_fft, int hop) {
    p.T = n_samples; p.n = n_fft; p.hop = hop;
    p.K = min(kBins, n_fft / 2 + 1);
    p.pad_left = (n_fft - hop) / 2;
    int pad_right = (n_fft - hop + 1) / 2;
    if (n_fft - n_samples - p.pad_left > pad_right) pad_right = n_fft - n_samples - p.pad_left;
    p.reflect = pad_right < n_samples ? 1 : 0;                  // then pad_left <= pad_right < n_samples as well
    p.n_frames = b2d_mel_frames(n_samples, n_fft, n_fft, hop);
    return p.n_frames;
}

// ---- backward: dL/dy for g = dL/dmel [B, n_mels, n_frames] (any element strides) ----
// Per frame f (Z = rfft of the windowed padded frame, mag and M = basis @ mag recomputed exactly as the forward):
//   gM[m]   = g[m, f] / M[m] where M[m] >= clip (torch's clamp(min=) passes the gradient at equality), else 0
//   gmag[k] = sum_m basis[m, k] gM[m]               (bin k: filters [bin_range[k][0], bin_range[k][1]), host-computed)
//   G[k]    = gmag[k] Z[k] / mag[k]                 (dL/dRe Z + j dL/dIm Z)
//   d[n]    = sum_{k=0..1024} Re(G[k] e^{+2 pi i k n / N})      (adjoint of the one-sided rfft)
//   dy_pad[f hop + n] += w[n] d[n];  padded index p -> src = p - pad_left, folded back by the reflection
//                                    (src < 0 -> -src, src >= T -> 2(T-1) - src) or dropped (constant padding)
// Frames are paired as in the forward ((2i, 2i+1) in one complex FFT, a lone last frame), so the recomputed M is
// bit-identical to the forward's.  The adjoint of the two frames is one more complex FFT: the Hermitian extensions
// H_a, H_b of G_a, G_b are packed as H_a + j H_b, and sum_k H[k] e^{+2 pi i k n / N} = FFT(H)[(N - n) mod N] returns
// d_a + j d_b.  Two FFTs per frame.
// Ownership: one CTA owns the waveform samples [s0, s0 + chunk) of one utterance and walks every frame that touches
// them (the halo frames are recomputed by both neighbours), including the frames whose reflected padding lands in
// them.  acc[] lives in shared memory; sample s0 + i belongs to thread i % 128 and gathers its terms frame by frame
// (direct, then left reflection, then right reflection): no atomics, and every sample is summed in a fixed order
// whatever the chunking, so the result is bitwise deterministic.
struct MelBwdParams {
    const float* y; const float* window; const float* basis;
    const int* lohi;           // [n_mels, 2]
    const int* bin_range;      // [1025, 2] first / one-past-last filter that is non-zero at each bin
    const float* g;            // dL/dmel, element (b, m, f) at g[b gs_b + m gs_m + f gs_f]
    long long gs_b, gs_m, gs_f;
    float* dy;                 // [B, T]
    int T, hop, n_frames, n_mels, pad_left, reflect, chunk;
    float clip;
};

constexpr int kMaxChunk = 8192;                              // samples per CTA at most (hop <= 4096)
constexpr size_t kBwdSmemFixed = (size_t)kPad * sizeof(float2) + (size_t)(kTw2 + kTw3) * sizeof(float2) +
                                 (size_t)2 * kMagStride * sizeof(float) + (size_t)2 * 128 * sizeof(float);

__device__ __forceinline__ int floordiv(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// acc[r - s0] += window[n] * d(n) for r in [rlo, rhi) owned by this thread, n = nof(r)
template <class NOf, class DOf>
__device__ __forceinline__ void gather_range(float* acc, int s0, int rlo, int rhi, const float* __restrict__ window,
                                             int tid, NOf nof, DOf dof) {
    if (rlo >= rhi) return;
    const int ilo = rlo - s0;
    for (int i = ilo + ((tid - ilo) % kThreads + kThreads) % kThreads; i < rhi - s0; i += kThreads) {
        const int n = nof(i + s0);
        acc[i] = fmaf(__ldg(window + n), dof(n), acc[i]);
    }
}

__global__ void __launch_bounds__(kThreads, 3) mel_bwd_kernel(MelBwdParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* F = reinterpret_cast<float2*>(smem_raw);
    float2* tw2 = F + kPad;
    float2* tw3 = tw2 + kTw2;
    float* mag = reinterpret_cast<float*>(tw3 + kTw3);        // [2][kMagStride]
    float* gm = mag + 2 * kMagStride;                         // [2][128]  gM of frames a, b
    float* acc = gm + 2 * 128;                                // [chunk]   dL/dy of the owned samples
    const int tid = threadIdx.x, b = blockIdx.y;
    const int T = p.T, hop = p.hop, pad_left = p.pad_left, nF = p.n_frames;
    const int s0 = blockIdx.x * p.chunk, s1 = min(s0 + p.chunk, T);
    const float* y = p.y + (size_t)b * T;
    const float* gb = p.g + (long long)b * p.gs_b + (long long)min(tid, p.n_mels - 1) * p.gs_m;

    b2d_fft_smem::init_twiddles<kN>(tw2, tw3, tid);
    int lo = 0, hi = 0;
    if (tid < p.n_mels) { lo = p.lohi[2 * tid]; hi = p.lohi[2 * tid + 1]; }
    const float* brow = p.basis + (size_t)min(tid, p.n_mels - 1) * kBins;
    for (int i = tid; i < s1 - s0; i += kThreads) acc[i] = 0.f;

    // ---- frames touching [s0, s1): directly, or through the reflected padding at either end ----
    int fl = max(0, floordiv(s0 + pad_left - kN, hop) + 1);
    int fh = min(nF - 1, floordiv(s1 - 1 + pad_left, hop));
    if (p.reflect) {
        const int rl = max(s0, 1);                            // left zone: r in [1, pad_left] <- src = -r
        if (rl <= pad_left && rl < s1) { fl = 0; fh = max(fh, min(nF - 1, (pad_left - rl) / hop)); }
        const int emax = (nF - 1) * hop - pad_left + kN - 1;  // right zone: r in [2(T-1) - emax, T-2] <- src = 2(T-1) - r
        const int rh = min(s1, T - 1);
        if (s0 <= T - 2 && rh - 1 >= 2 * (T - 1) - emax) {
            const int need = 2 * T - kN - rh + pad_left;      // a frame reaches r = rh - 1 once f hop >= need
            fl = min(fl, max(0, need <= 0 ? 0 : (need + hop - 1) / hop));
            fh = nF - 1;
        }
    }
    __syncthreads();

    for (int fa = fl & ~1; fa <= fh; fa += 2) {
        const bool has_b = fa + 1 < nF;
        float ga = 0.f, gbv = 0.f;                            // cotangents, in flight across the FFT
        if (tid < p.n_mels) {
            ga = __ldg(gb + (long long)fa * p.gs_f);
            if (has_b) gbv = __ldg(gb + (long long)(fa + 1) * p.gs_f);
        }
        // ---- forward recomputation: Z, mag, M of frames fa and fa + 1 ----
        load_frame_pair(F, y, p.window, T, hop, pad_left, p.reflect, fa, has_b, tid);
        __syncthreads();
        b2d_fft_smem::fft_forward<kN, 1, true>(F, tw2, tw3, tid);
        pair_magnitudes(F, mag, tid);
        __syncthreads();
        if (tid < p.n_mels) {
            float sa, sb;
            project_pair(mag, brow, lo, hi, sa, sb);
            gm[tid] = sa >= p.clip ? ga / sa : 0.f;           // d log(max(M, clip)) / dM
            gm[128 + tid] = sb >= p.clip ? gbv / sb : 0.f;
        }
        __syncthreads();
        // ---- gmag, G and the packed Hermitian spectrum H_a + j H_b, in place (bin k also owns N - k) ----
        for (int k = tid; k < kBins; k += kThreads) {
            const int m0 = __ldg(p.bin_range + 2 * k), m1 = __ldg(p.bin_range + 2 * k + 1);
            float da = 0.f, db = 0.f;
            for (int m = m0; m < m1; ++m) {
                const float wgt = __ldg(p.basis + (size_t)m * kBins + k);
                da = fmaf(wgt, gm[m], da);
                db = fmaf(wgt, gm[128 + m], db);
            }
            float ar, ai, br, bi;
            split_pair(F, k, ar, ai, br, bi);
            const float ca = da / mag[k], cb = db / mag[kMagStride + k];
            const float gar = ca * ar, gai = ca * ai, gbr = cb * br, gbi = cb * bi;
            if (k == 0 || k == kN / 2) {
                F[padi(k)] = make_float2(gar, gbr);           // DC / Nyquist: Re(G e^{...}) keeps Re G only
            } else {
                F[padi(k)] = make_float2(0.5f * (gar - gbi), 0.5f * (gai + gbr));
                F[padi(kN - k)] = make_float2(0.5f * (gar + gbi), 0.5f * (gbr - gai));
            }
        }
        __syncthreads();
        b2d_fft_smem::fft_forward<kN, 1, true>(F, tw2, tw3, tid);
        // ---- overlap-add of w d into the owned samples, folding the padding back ----
#pragma unroll 1
        for (int which = 0; which < 2; ++which) {
            if (which == 1 && !has_b) break;
            const int A = (fa + which) * hop - pad_left;      // src of frame sample 0
            auto dof = [&](int n) { const float2 v = F[padi((kN - n) & (kN - 1))]; return which ? v.y : v.x; };
            gather_range(acc, s0, max(s0, A), min(s1, A + kN), p.window, tid, [&](int r) { return r - A; }, dof);
            if (p.reflect) {
                gather_range(acc, s0, max(max(s0, 1), -A - kN + 1), min(s1, -A + 1), p.window, tid,
                             [&](int r) { return -r - A; }, dof);
                const int m2 = 2 * (T - 1) - A;
                gather_range(acc, s0, max(s0, m2 - kN + 1), min(min(s1, T - 1), m2 + 1), p.window, tid,
                             [&](int r) { return m2 - r; }, dof);
            }
        }
        __syncthreads();                                      // F is rewritten by the next pair's loads
    }
    float* dy = p.dy + (size_t)b * T;
    for (int i = tid; i < s1 - s0; i += kThreads) dy[s0 + i] = acc[i];
}

}  // namespace

extern "C" int b2d_mel_frames(int n_samples, int n_fft, int win_size, int hop) {
    if (n_samples <= 0 || hop <= 0 || win_size < hop || n_fft < win_size) return 0;
    const int pad_left = (win_size - hop) / 2;
    int pad_right = (win_size - hop + 1) / 2;
    if (win_size - n_samples - pad_left > pad_right) pad_right = win_size - n_samples - pad_left;
    const long long padded = (long long)n_samples + pad_left + pad_right;
    return padded < n_fft ? 0 : (int)(1 + (padded - n_fft) / hop);
}

extern "C" int b2d_mel_keyshift_table_floats(int n_fft) {
    if (n_fft < 1 || n_fft > kKeyshiftMaxN) return 0;
    return bluestein_table_floats(n_fft, min(kBins, n_fft / 2 + 1));
}

#ifndef B2D_HOST_EMU

namespace {
template <int M, bool ZU> int launch_keyshift(const MelKeyshiftParams& p, int B, cudaStream_t st) {
    constexpr size_t smem = keyshift_smem_bytes<M>();
    cudaError_t e = cudaFuncSetAttribute(mel_keyshift_kernel<M, ZU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return b2d::fail((int)e, "mel_spectrogram_keyshift: smem attr: %s", cudaGetErrorString(e));
    mel_keyshift_kernel<M, ZU><<<dim3((p.n_frames + 1) / 2, B), kThreads, smem, st>>>(p);
    return b2d::check_launch("mel_spectrogram_keyshift");
}
}  // namespace

extern "C" int b2d_mel_spectrogram_keyshift(const float* audio, const float* table, const float* mel_basis,
                                            const int* filter_lohi, int B, int n_samples, int n_fft, int hop, int n_mels,
                                            float clip_val, float* mel, void* stream) {
    if (!audio || !table || !mel_basis || !filter_lohi || !mel)
        return b2d::fail(B2D_ERR_NULL, "mel_spectrogram_keyshift: null pointer");
    if ((uintptr_t)table & 7) return b2d::fail(B2D_ERR_ALIGN, "mel_spectrogram_keyshift: table not 8-byte aligned");
    if (B <= 0 || B > 65535 || n_samples <= 0 || hop <= 0 || n_mels <= 0 || n_mels > 128)
        return b2d::fail(B2D_ERR_SHAPE, "mel_spectrogram_keyshift: bad shape B=%d T=%d hop=%d n_mels=%d (n_mels <= 128)",
                         B, n_samples, hop, n_mels);
    if (n_fft < hop || n_fft > kKeyshiftMaxN)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "mel_spectrogram_keyshift: n_fft %d outside [hop = %d, %d]", n_fft, hop,
                         kKeyshiftMaxN);
    MelKeyshiftParams p;
    p.y = audio; p.table = table; p.basis = mel_basis; p.lohi = filter_lohi; p.out = mel;
    p.n_mels = n_mels; p.clip = clip_val;
    if (keyshift_setup(p, n_samples, n_fft, hop) <= 0)
        return b2d::fail(B2D_ERR_SHAPE, "mel_spectrogram_keyshift: signal too short");
    cudaStream_t st = (cudaStream_t)stream;
    const int M = bluestein_size(n_fft, p.K);
    const bool zu = 2 * n_fft <= M;
    if (M == 1024) return zu ? launch_keyshift<1024, true>(p, B, st) : launch_keyshift<1024, false>(p, B, st);
    if (M == 2048) return zu ? launch_keyshift<2048, true>(p, B, st) : launch_keyshift<2048, false>(p, B, st);
    return zu ? launch_keyshift<4096, true>(p, B, st) : launch_keyshift<4096, false>(p, B, st);
}

extern "C" int b2d_mel_spectrogram(const float* audio, const float* window, const float* mel_basis, const int* filter_lohi,
                                   int B, int n_samples, int n_fft, int win_size, int hop, int n_mels, float clip_val,
                                   float* mel, void* stream) {
    if (!audio || !window || !mel_basis || !filter_lohi || !mel) return b2d::fail(B2D_ERR_NULL, "mel_spectrogram: null pointer");
    if (n_fft != kN || win_size != kN)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "mel_spectrogram: only n_fft = win_size = %d is built (keyshift 0), got %d / %d", kN, n_fft, win_size);
    if (B <= 0 || B > 65535 || n_samples <= 0 || hop <= 0 || hop > kN || n_mels <= 0 || n_mels > 128)
        return b2d::fail(B2D_ERR_SHAPE, "mel_spectrogram: bad shape B=%d T=%d hop=%d n_mels=%d (n_mels <= 128)", B, n_samples, hop, n_mels);
    MelParams p;
    p.y = audio; p.window = window; p.basis = mel_basis; p.lohi = filter_lohi; p.out = mel;
    p.T = n_samples; p.hop = hop; p.n_mels = n_mels; p.clip = clip_val;
    p.pad_left = (win_size - hop) / 2;
    int pad_right = (win_size - hop + 1) / 2;
    if (win_size - n_samples - p.pad_left > pad_right) pad_right = win_size - n_samples - p.pad_left;
    p.reflect = pad_right < n_samples ? 1 : 0;                  // nvSTFT.py:99-102
    if (p.reflect && (p.pad_left >= n_samples || pad_right >= n_samples))
        return b2d::fail(B2D_ERR_SHAPE, "mel_spectrogram: reflect padding needs more than %d samples", p.pad_left);
    p.n_frames = b2d_mel_frames(n_samples, n_fft, win_size, hop);
    if (p.n_frames <= 0) return b2d::fail(B2D_ERR_SHAPE, "mel_spectrogram: signal too short");
    cudaError_t e = cudaFuncSetAttribute(mel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
    if (e != cudaSuccess) return b2d::fail((int)e, "mel_spectrogram: smem attr: %s", cudaGetErrorString(e));
    dim3 grid((p.n_frames + kFramesPerCta - 1) / kFramesPerCta, B);
    mel_kernel<<<grid, kThreads, kSmemBytes, (cudaStream_t)stream>>>(p);
    return b2d::check_launch("mel_spectrogram");
}

extern "C" int b2d_mel_spectrogram_backward(const float* audio, const float* window, const float* mel_basis,
                                            const int* filter_lohi, const int* bin_filter_range, int B, int n_samples,
                                            int n_fft, int win_size, int hop, int n_mels, float clip_val,
                                            const float* grad_mel, int64_t grad_stride_b, int64_t grad_stride_mel,
                                            int64_t grad_stride_frame, float* grad_audio, void* stream) {
    if (!audio || !window || !mel_basis || !filter_lohi || !bin_filter_range || !grad_mel || !grad_audio)
        return b2d::fail(B2D_ERR_NULL, "mel_spectrogram_backward: null pointer");
    if (n_fft != kN || win_size != kN)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "mel_spectrogram_backward: only n_fft = win_size = %d is built (keyshift 0), "
                         "got %d / %d", kN, n_fft, win_size);
    if (B <= 0 || B > 65535 || n_samples <= 0 || hop <= 0 || hop > kN || n_mels <= 0 || n_mels > 128)
        return b2d::fail(B2D_ERR_SHAPE, "mel_spectrogram_backward: bad shape B=%d T=%d hop=%d n_mels=%d (n_mels <= 128)",
                         B, n_samples, hop, n_mels);
    if (grad_stride_b < 0 || grad_stride_mel < 0 || grad_stride_frame < 0)
        return b2d::fail(B2D_ERR_SHAPE, "mel_spectrogram_backward: negative grad_mel stride");
    MelBwdParams p;
    p.y = audio; p.window = window; p.basis = mel_basis; p.lohi = filter_lohi; p.bin_range = bin_filter_range;
    p.g = grad_mel; p.gs_b = grad_stride_b; p.gs_m = grad_stride_mel; p.gs_f = grad_stride_frame; p.dy = grad_audio;
    p.T = n_samples; p.hop = hop; p.n_mels = n_mels; p.clip = clip_val;
    p.pad_left = (win_size - hop) / 2;
    int pad_right = (win_size - hop + 1) / 2;
    if (win_size - n_samples - p.pad_left > pad_right) pad_right = win_size - n_samples - p.pad_left;
    p.reflect = pad_right < n_samples ? 1 : 0;
    if (p.reflect && (p.pad_left >= n_samples || pad_right >= n_samples))
        return b2d::fail(B2D_ERR_SHAPE, "mel_spectrogram_backward: reflect padding needs more than %d samples", p.pad_left);
    p.n_frames = b2d_mel_frames(n_samples, n_fft, win_size, hop);
    if (p.n_frames <= 0) return b2d::fail(B2D_ERR_SHAPE, "mel_spectrogram_backward: signal too short");
    // chunk: an even number of hops, at most kMaxChunk samples (a chunk of H hops walks about H + 4 frames); shrink it
    // while the grid would hold fewer than 4 CTAs per SM
    int hops = max(2, 2 * (kMaxChunk / (2 * hop)));
    while (hops > 2 && (long long)B * ((n_samples + hops * hop - 1) / (hops * hop)) < 4LL * b2d::num_sms()) hops -= 2;
    p.chunk = hops * hop;
    const size_t smem = kBwdSmemFixed + (size_t)p.chunk * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(mel_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)(kBwdSmemFixed + (size_t)kMaxChunk * sizeof(float)));
    if (e != cudaSuccess) return b2d::fail((int)e, "mel_spectrogram_backward: smem attr: %s", cudaGetErrorString(e));
    dim3 grid((n_samples + p.chunk - 1) / p.chunk, B);
    mel_bwd_kernel<<<grid, kThreads, smem, (cudaStream_t)stream>>>(p);
    return b2d::check_launch("mel_spectrogram_backward");
}
#endif  // B2D_HOST_EMU
