// Backward of the old CombSub synthesizer (api.cu b2d_combsub_synth) with respect to its three raw controls, for the
// training phase (infer=False): reference ddsp/vocoder.py:834-862, ddsp/core.py:120-182,240-270.  See DESIGN §4.5b.
//
// The forward chain is a = FIR(comb, h_ap), harmonic = FIR(a, h_h), noise = FIR(u, h_n), in the direct form of
// sins_bwd.cu (h_nF := h_{nF-1}).  With g_h = dL/dsignal + dL/dharmonic and g_n = dL/dsignal + dL/dnoise:
//   combsub_bwd_kernel, stage 1, one CTA per (frame f, utterance):
//       harmonic filter: dh_h = corr(g_h, allpassed); da = FIR^T(g_h, h_h) for hop f (the cascade's input gradient,
//       written to the backward workspace); un-roll dh_h, times this frame's dynamic window (the fp32 formula of
//       ir_build_tc.cu), adjoint of torch's c2r irfft, dc_h = Re(dH) exp(c_h);
//       noise filter: dh_n = corr(g_n, u) with u regenerated (or noise_in), Hann, irfft adjoint, dc_n = Re(dH) exp(c)/128;
//   combsub_bwd_kernel, stage 2 (needs da of hops f-1 .. f+1 and the tap overhang, so a second launch):
//       all-pass filter: dh_ap = corr(da, comb), irfft adjoint, dphi_j = Im(dH_j conj H_j), reverse cumsum,
//       * pi (1 - tanh^2 c).  No input gradient: the comb depends on f0 only, which is data.
// Up to 1024 taps (n_mag <= 513): a thread owns taps 4 t .. 4 t + 3 and 512 + 4 t .. 512 + 4 t + 3.
// Every gradient element and every da sample has exactly one owning thread, which sums its terms in a fixed order: no
// atomics, results independent of the grid, of b2d_set_overlap and of batch sharding (the noise is keyed by the global
// utterance index).
#ifndef B2D_HOST_EMU               // tests/emu/ runs these kernels' source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif
#include "fir_adjoint.cuh"

namespace {

constexpr int kP = 512;                      // block size the backward is built for
constexpr int kMaxTaps = 1024;               // 2 (n_mag - 1), n_mag <= 513
constexpr int kMaxBins = kMaxTaps / 2 + 1;
constexpr int kThreads = 128;
constexpr int kWin = 2 * kP + kMaxTaps + 4;  // cotangent window of one frame (+ the register window's overhang)
using b2d_firadj::kSub;

enum Filter { kAllpass = 0, kHarmonic = 1, kNoise = 2 };

struct CsBwdParams {
    const float* comb;        // [B, T] the forward's comb source
    const float* allpassed;   // [B, T] the forward's all-pass output
    const float* noise_in;    // [B, T] or nullptr: in-kernel Philox noise keyed by (seed, utt_off + b)
    unsigned long long seed;
    long long utt_off;
    const float* ir_h;        // [B, nF, Lh] the forward's harmonic impulse responses
    const float* f0;          // [B, nF] (dynamic window)
    float hw_num;             // 1.5 sr in fp32, as ir_build.cu
    const float* c_gd;        // raw controls, frame stride ctrl_stride
    const float* c_hm;
    const float* c_nm;
    long long ctrl_stride;
    const float* g;           // dL/dsignal, dL/dharmonic, dL/dnoise [B, T] (nullptr = zero)
    const float* g_harm;
    const float* g_noise;
    int nF, Ma, Mh, Mn;
    float* da;                // [B, T] dL/dallpassed (stage 1 writes it, stage 2 reads it)
    float* grad;              // dense [B, nF, Ma + Mh + Mn]
};

struct CsSmem {
    float gw[kWin];                    // cotangent window, origin at sample (f-1)P - L/2
    float v[2 * kP];                   // weighted filter input of hops f-1, f
    float hA[kMaxTaps], hB[kMaxTaps];  // h_f, h_{f+1} of the harmonic filter, zero-padded
    float dh[kMaxTaps];
    float cosT[kMaxTaps], sinT[kMaxTaps];   // cos / sin(2 pi t / N)
    float2 eo[kMaxTaps / 2];           // (dr[n] + dr[N-n], dr[n] - dr[N-n]) for 1 <= n < N/2, zero elsewhere
    float d0, dN;                      // dr[0], dr[N/2]
    float tmp[kMaxBins + 3];
    double cum[kMaxBins + 3];
    double part[2 * kThreads];
};

__device__ void filter_bwd(const CsBwdParams& p, CsSmem& s, Filter which) {
    const int f = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int nF = p.nF;
    const long long T = (long long)nF * kP;
    const size_t row = (size_t)b * (size_t)T;
    const size_t frow = (size_t)b * nF + f;
    float* grow = p.grad + frow * (size_t)(p.Ma + p.Mh + p.Mn);
    const bool ap = which == kAllpass, harm = which == kHarmonic;
    const int M = ap ? p.Ma : harm ? p.Mh : p.Mn, L = 2 * (M - 1), N = L, half = L / 2;
    const float* g1 = ap ? p.da : p.g;
    const float* g2 = ap ? nullptr : harm ? p.g_harm : p.g_noise;
    const float* crow = (ap ? p.c_gd : harm ? p.c_hm : p.c_nm) + frow * (size_t)p.ctrl_stride;
    const long long n0 = (long long)(f - 1) * kP - half;

    // ---- stage: cotangent window, weighted input, filter rows, DFT table, raw activations ----
    for (int i = tid; i < kWin; i += kThreads) {
        const long long n = n0 + i;
        float v = 0.f;
        if (i < 2 * kP + L - 1 && n >= 0 && n < T) {
            if (g1) v = g1[row + n];
            if (g2) v += g2[row + n];
        }
        s.gw[i] = v;
    }
    for (int q = tid; q < 2 * kP / 4; q += kThreads) {
        const int i = 4 * q;
        const long long m = (long long)(f - 1) * kP + i;
        float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m >= 0 && m < T) {          // whole quads: m and T are multiples of 4
            if (ap) x = *reinterpret_cast<const float4*>(p.comb + row + m);
            else if (harm) x = *reinterpret_cast<const float4*>(p.allpassed + row + m);
            else if (p.noise_in) x = *reinterpret_cast<const float4*>(p.noise_in + row + m);
            else x = b2d::philox_uniform_pm1(p.seed, (unsigned long long)(p.utt_off + b), (uint32_t)(m >> 2));
        }
        const float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int ii = i + k;
            float w;
            if (ii < kP) w = (float)ii * (1.0f / kP);                                  // hop f-1: phi
            else w = (f == nF - 1) ? 1.0f : 1.0f - (float)(ii - kP) * (1.0f / kP);    // hop f: 1 - phi (+ held row)
            s.v[ii] = w * xs[k];
        }
    }
    if (harm) {
        const float* ir = p.ir_h + (size_t)b * nF * L;
        const int f1 = min(f + 1, nF - 1);
        for (int t = tid; t < kMaxTaps; t += kThreads) {
            s.hA[t] = t < L ? ir[(size_t)f * L + t] : 0.f;
            s.hB[t] = t < L ? ir[(size_t)f1 * L + t] : 0.f;
        }
    }
    for (int t = tid; t < N; t += kThreads) {
        double sd, cd;
        sincospi(2.0 * (double)t / (double)N, &sd, &cd);
        s.cosT[t] = (float)cd;
        s.sinT[t] = (float)sd;
    }
    if (ap)
        for (int j = tid; j < M; j += kThreads) s.tmp[j] = B2D_PI_F * tanhf(crow[j]);   // the forward's pi tanh(c)
    __syncthreads();

    // ---- dh: thread owns taps 4 t4 .. 4 t4 + 3 for t4 = tid, tid + 128 ----
#pragma unroll 1
    for (int grp = 0; grp < kMaxTaps / (4 * kThreads); ++grp) {
        const int t4 = tid + grp * kThreads;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        if (4 * t4 < L) b2d_firadj::corr4(s.gw, s.v, t4, 2 * kP / 4, acc);
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (4 * t4 + k < L) s.dh[4 * t4 + k] = acc[k];
    }
    // ---- da of hop f (harmonic filter only): thread owns samples 4 tid .. 4 tid + 3 ----
    if (harm) {
        float a[4] = {0.f, 0.f, 0.f, 0.f}, c[4] = {0.f, 0.f, 0.f, 0.f};
        b2d_firadj::fir_t4(s.gw + kP, s.hA, s.hB, tid, (L + 3) / 4, a, c);
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float ph = (float)(4 * tid + k) * (1.0f / kP);
            o[k] = fmaf(1.0f - ph, a[k], ph * c[k]);
        }
        *reinterpret_cast<float4*>(p.da + row + (size_t)f * kP + 4 * tid) = make_float4(o[0], o[1], o[2], o[3]);
    }
    if (ap) b2d_firadj::block_scan<kThreads>(s.tmp, s.cum, M, false, s.part);   // forward phase phi_j (barrier)
    else __syncthreads();

    // ---- un-roll the causal form: dr[n] = dh[(n + L/2) mod L] times the window of that tap ----
    const float hw = harm ? p.hw_num / (p.f0[frow] + 1e-3f) : 1.f;
    auto dr = [&](int n) -> float {
        int t = n + half;
        if (t >= L) t -= L;
        const float v = s.dh[t];
        if (ap) return v;
        if (!harm) return v * (0.5f - 0.5f * s.cosT[t]);                 // periodic Hann
        float u = (float)(t - (M - 1)) / hw;                             // dynamic raised cosine, ir_build_tc.cu's
        if (u > 1.f) u = 0.f;                                            // formula: cos(pi u) by exact period
        const float r = fmaf(-2.0f, rintf(0.5f * u), u);                 // reduction (cosf's large-argument path
        return v * ((1.f + __cosf(B2D_PI_F * r)) * 0.5f);                // would put a stack frame here)
    };
    for (int n = tid; n < kMaxTaps / 2; n += kThreads) {
        float2 e = make_float2(0.f, 0.f);
        if (n >= 1 && n < half) {
            const float lo = dr(n), hi = dr(N - n);
            e = make_float2(lo + hi, lo - hi);
        }
        s.eo[n] = e;
    }
    if (tid == 0) { s.d0 = dr(0); s.dN = dr(half); }
    __syncthreads();

    // ---- adjoint of irfft per bin, then the activation ----
    const int nblk = (half + kSub - 1) / kSub;
    for (int j = tid; j < M; j += kThreads) {
        float dre, dim;
        b2d_firadj::irfft_adjoint_bin(j, M, N, nblk, s.cosT, s.sinT, s.eo, s.d0, s.dN, dre, dim);
        if (ap) {
            float sn, cs;
            sincosf((float)s.cum[j], &sn, &cs);
            s.tmp[j] = dim * cs - dre * sn;                    // dphi_j = Im(dH conj(H))
        } else if (harm) {
            grow[p.Ma + j] = dre * expf(crow[j]);
        } else {
            grow[p.Ma + p.Mh + j] = (dre * 0.0078125f) * expf(crow[j]);
        }
    }
    if (ap) {
        __syncthreads();
        b2d_firadj::block_scan<kThreads>(s.tmp, s.cum, M, true, s.part);    // reverse cumsum: sum_{i >= j} dphi_i
        for (int j = tid; j < M; j += kThreads) {
            const float th = tanhf(crow[j]);
            grow[j] = ((float)s.cum[j] * B2D_PI_F) * (1.0f - th * th);
        }
    }
    __syncthreads();   // the next filter restages every buffer
}

// stage 1: harmonic filter (dh_h, da) and noise filter; stage 2: all-pass filter on da
template <int STAGE>
__global__ void __launch_bounds__(kThreads) combsub_bwd_kernel(CsBwdParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    CsSmem& s = *reinterpret_cast<CsSmem*>(smem_raw);
    if (STAGE == 1) {
        filter_bwd(p, s, kHarmonic);
        filter_bwd(p, s, kNoise);
    } else {
        filter_bwd(p, s, kAllpass);
    }
}

}  // namespace

#ifndef B2D_HOST_EMU
namespace {
inline size_t align256(size_t v) { return (v + 255) / 256 * 256; }

template <int STAGE>
int stage_launch(const CsBwdParams& p, int B, cudaStream_t st) {
    auto kern = combsub_bwd_kernel<STAGE>;
    if (sizeof(CsSmem) > 48 * 1024) {
        const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(CsSmem));
        if (e != cudaSuccess) return b2d::fail((int)e, "combsub_synth_backward: smem attr: %s", cudaGetErrorString(e));
    }
    kern<<<dim3((unsigned)p.nF, (unsigned)B), kThreads, sizeof(CsSmem), st>>>(p);
    return b2d::check_launch(STAGE == 1 ? "combsub_synth_backward: stage 1" : "combsub_synth_backward: stage 2");
}
}  // namespace

extern "C" size_t b2d_combsub_synth_backward_workspace_bytes(int B, int n_frames, int block) {
    if (B <= 0 || n_frames <= 0 || block <= 0) return 0;
    return align256((size_t)B * n_frames * block * 4);     // dL/dallpassed
}

extern "C" int b2d_combsub_synth_backward(const float* f0_frames, const float* c_group_delay, const float* c_harmonic,
                                          const float* c_noise, int64_t ctrl_stride, const float* noise_in,
                                          uint64_t seed, int64_t utterance_offset, const void* forward_workspace,
                                          const float* grad_signal, const float* grad_harmonic,
                                          const float* grad_noise, int B, int n_frames, int block, int n_mag_allpass,
                                          int n_mag_harmonic, int n_mag_noise, double sampling_rate, float* grad_ctrl,
                                          void* workspace, size_t workspace_bytes, void* stream) {
    if (!f0_frames || !c_group_delay || !c_harmonic || !c_noise || !forward_workspace || !grad_ctrl || !workspace)
        return b2d::fail(B2D_ERR_NULL, "combsub_synth_backward: null pointer");
    if (B <= 0 || n_frames <= 0 || block <= 0 || n_mag_allpass < 2 || n_mag_harmonic < 2 || n_mag_noise < 2 ||
        ctrl_stride < n_mag_allpass || ctrl_stride < n_mag_harmonic || ctrl_stride < n_mag_noise)
        return b2d::fail(B2D_ERR_SHAPE, "combsub_synth_backward: bad shape B=%d nF=%d block=%d Ma=%d Mh=%d Mn=%d "
                         "stride=%lld", B, n_frames, block, n_mag_allpass, n_mag_harmonic, n_mag_noise,
                         (long long)ctrl_stride);
    if (block != kP || n_mag_allpass > kMaxBins || n_mag_harmonic > kMaxBins || n_mag_noise > kMaxBins || B > 65535)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "combsub_synth_backward: built for block %d, n_mag <= %d, B <= 65535 "
                         "(got block %d, n_mag %d / %d / %d, B %d)", kP, kMaxBins, block, n_mag_allpass,
                         n_mag_harmonic, n_mag_noise, B);
    const size_t need = b2d_combsub_synth_backward_workspace_bytes(B, n_frames, block);
    if (workspace_bytes < need)
        return b2d::fail(B2D_ERR_WORKSPACE, "combsub_synth_backward: workspace %zu < %zu bytes", workspace_bytes, need);
    if ((reinterpret_cast<uintptr_t>(workspace) & 255u) || (reinterpret_cast<uintptr_t>(forward_workspace) & 255u) ||
        (noise_in && !b2d::aligned16(noise_in)) || (reinterpret_cast<uintptr_t>(grad_ctrl) & 3u))
        return b2d::fail(B2D_ERR_ALIGN, "combsub_synth_backward: workspaces must be 256-byte aligned, noise_in 16-byte "
                         "aligned");

    // forward workspace (api.cu b2d_combsub_synth): comb | allpassed | noise | ir_ap | ir_h | ir_n
    const size_t BT = (size_t)B * n_frames * block, BF = (size_t)B * n_frames;
    const size_t sBT = align256(BT * 4);
    const int La = 2 * (n_mag_allpass - 1);
    const char* fws = static_cast<const char*>(forward_workspace);
    CsBwdParams p;
    p.comb = reinterpret_cast<const float*>(fws);
    p.allpassed = reinterpret_cast<const float*>(fws + sBT);
    p.ir_h = reinterpret_cast<const float*>(fws + 3 * sBT + align256(BF * La * 4));
    p.noise_in = noise_in; p.seed = seed; p.utt_off = utterance_offset;
    p.f0 = f0_frames; p.hw_num = 1.5f * (float)sampling_rate;
    p.c_gd = c_group_delay; p.c_hm = c_harmonic; p.c_nm = c_noise; p.ctrl_stride = ctrl_stride;
    p.g = grad_signal; p.g_harm = grad_harmonic; p.g_noise = grad_noise;
    p.nF = n_frames; p.Ma = n_mag_allpass; p.Mh = n_mag_harmonic; p.Mn = n_mag_noise;
    p.da = static_cast<float*>(workspace); p.grad = grad_ctrl;
    cudaStream_t st = (cudaStream_t)stream;
    const int rc = stage_launch<1>(p, B, st);
    if (rc) return rc;
    return stage_launch<2>(p, B, st);
}
#endif  // B2D_HOST_EMU
