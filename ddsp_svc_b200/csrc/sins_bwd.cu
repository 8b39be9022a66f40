// Backward of the Sins synthesizer (api.cu b2d_sins_synth) with respect to its three raw controls, for the training
// phase (infer=False): reference ddsp/vocoder.py:580-611, ddsp/core.py:66-77,120-182,254-270.  See DESIGN §4.4c.
//
// With g_h = dL/dsignal + dL/dharmonic and g_n = dL/dsignal + dL/dnoise, and the direct form of the time-varying FIR
//   y[n] = sum_tau ((1 - phi_m) h_f[tau] + phi_m h_{f+1}[tau]) x[m],  m = n + L/2 - tau, f = m / P, phi_m = (m mod P)/P,
// (h_nF := h_{nF-1}), the two kernels below compute
//   sins_fir_bwd_kernel   one CTA per (frame f, utterance):
//       dh_f[tau] = sum_{i < 2P} v[i] g[(f-1)P + i - L/2 + tau],  v = x weighted by phi (hop f-1) and 1 - phi (hop f; 1 at
//                   the last row, which also carries the held row nF) -- for both filters (x = sinusoids / the noise);
//       dx[fP + q] = (1 - phi) sum_tau h_f[tau] g_h[fP + q - L/2 + tau] + phi sum_tau h_{f+1}[tau] g_h[...];
//       the impulse-response adjoints: un-roll dh, adjoint of torch's c2r irfft (1/N at DC and Nyquist, whose imaginary
//       part irfft drops, 2/N elsewhere), then all-pass dphi_j = Im(dH_j conj(H_j)), reverse cumsum, * pi (1 - tanh^2 c);
//       noise: Hann window first, dc = Re(dH) exp(c)/128;
//   sins_bank_bwd_kernel  one CTA per (frame k, utterance):
//       dA[k,h] = sum_t dx(t) sin(h phi(t)) w_k(t) over hops k-1, k (w_k the linear-upsample hat; weight 1 on hop k at the
//       last row), dc = dA * A, A = exp(c)/128 * (1[f0 h < sr/2] + 1e-7); the phase is the forward's (sample_phase with
//       the infer=False per-sample fp32 rounding).
// Every gradient element and every dx sample has exactly one owning thread, which sums its terms in a fixed order: no
// atomics, results independent of the grid, of b2d_set_overlap and of b2d_set_sins_impl.
#ifndef B2D_HOST_EMU               // tests/emu/ runs these kernels' source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif
#include "fir_adjoint.cuh"
#include "sins_bank_math.cuh"

namespace {

using b2d_firadj::kP;                        // block size the backward is built for
using b2d_firadj::kThreads;
constexpr int kMaxTaps = 512;                // 2 (n_mag - 1), n_mag <= 257
constexpr int kMaxBins = kMaxTaps / 2 + 1;

struct FirBwdParams {
    const float* sinus;       // [B, T] the forward's oscillator-bank output
    const float* noise_in;    // [B, T] or nullptr: in-kernel Philox noise keyed by (seed, utt_off + b)
    unsigned long long seed;
    long long utt_off;
    const float* ir_ap;       // [B, nF, La]
    const float* ir_n;        // [B, nF, Ln]
    const float* c_gd;        // raw group_delay / noise_magnitude controls, frame stride ctrl_stride
    const float* c_nm;
    long long ctrl_stride;
    const float* g;           // dL/dsignal, dL/dharmonic, dL/dnoise [B, T] (nullptr = zero)
    const float* g_harm;
    const float* g_noise;
    int nF, Ma, Mn, H;
    float* dx;                // [B, T] dL/dsinusoids
    float* grad;              // dense [B, nF, H + Ma + Mn]
};

using FirSmem = b2d_firadj::FirSmem<kMaxTaps>;

__global__ void __launch_bounds__(kThreads) sins_fir_bwd_kernel(FirBwdParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    FirSmem& s = *reinterpret_cast<FirSmem*>(smem_raw);
    const size_t frow = (size_t)blockIdx.y * p.nF + blockIdx.x;
    float* grow = p.grad + frow * (size_t)(p.H + p.Ma + p.Mn);
    b2d_firadj::FirArgs a{};
    a.nF = p.nF; a.seed = p.seed; a.utt_off = p.utt_off; a.grad_row = grow; a.g = p.g;

    a.M = p.Ma; a.x = p.sinus; a.g_add = p.g_harm; a.ir = p.ir_ap; a.dx = p.dx;
    a.ctrl = p.c_gd + frow * (size_t)p.ctrl_stride; a.col = p.H;
    b2d_firadj::fir_adjoint<b2d_firadj::kAllpass>(s, a);

    a.M = p.Mn; a.x = p.noise_in; a.g_add = p.g_noise; a.ir = nullptr; a.dx = nullptr;
    a.ctrl = p.c_nm + frow * (size_t)p.ctrl_stride; a.col = p.H + p.Ma;
    b2d_firadj::fir_adjoint<b2d_firadj::kNoise>(s, a);
}

// ---------------------------------------------------------------------------------------------------------------------
constexpr int kTile = 128;                   // samples per staged tile
constexpr int kSlices = kThreads / b2d_bank::kNA;   // 8 sample slices x 16 anchors
constexpr int kBaseStride = 33;              // float2 per staged sample (<= 32 bases + 1 against bank conflicts)

struct BankBwdParams {
    const float* f0;
    const double* frame_phase;
    const float* c_amp;
    long long ctrl_stride;
    const float* dx;
    int nF, H;
    double inv_sr;
    float nyquist;
    float* grad;                 // dense [B, nF, H + Ma + Mn]
    long long grad_stride;
};

struct BankSmem {
    float x32[kTile];
    float u[kTile];
    float2 base[kTile * kBaseStride];        // (cos, sin) of base harmonic hb = 128 g + 16 b; reused for the reduction
};

template <int G>
__global__ void __launch_bounds__(kThreads) sins_bank_bwd_kernel(BankBwdParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    BankSmem& s = *reinterpret_cast<BankSmem*>(smem_raw);
    const int k = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int nF = p.nF;
    const int a = tid % b2d_bank::kNA, sl = tid / b2d_bank::kNA;
    const float af = (float)(a + 1);
    const size_t row = (size_t)b * nF * kP;
    constexpr int NBASE = 8 * G;
    float acc[NBASE];
#pragma unroll
    for (int i = 0; i < NBASE; ++i) acc[i] = 0.f;

    for (int i0 = 0; i0 < 2 * kP; i0 += kTile) {
        {
            const int i = i0 + tid;
            const int hop = i < kP ? k - 1 : k, j = i < kP ? i : i - kP;
            float x = 0.f, u = 0.f;
            if (hop >= 0) {
                const size_t fr = (size_t)b * nF + hop;
                const double fk = (double)p.f0[fr];
                const double dk = (double)p.f0[(size_t)b * nF + min(hop + 1, nF - 1)] - fk;
                x = b2d_bank::sample_phase(p.frame_phase[fr], fk, dk, j, 0.5 / (double)kP, p.inv_sr, 1);
                const float w = i < kP ? (float)j * (1.0f / kP) : (k == nF - 1 ? 1.0f : 1.0f - (float)j * (1.0f / kP));
                u = p.dx[row + (size_t)hop * kP + j] * w;
            }
            s.x32[tid] = x;
            s.u[tid] = u;
        }
        __syncthreads();
        for (int e = tid; e < kTile * NBASE; e += kThreads) {
            const int i = e / NBASE, gb = e - i * NBASE;
            const float hb = (float)(128 * (gb >> 3) + 16 * (gb & 7));
            const float x = s.x32[i];
            const float r = fmaf(hb, x, -rintf(hb * x));      // exactly reduced, as the forward's base rotation
            float sn, cs;
            __sincosf(B2D_TWO_PI_F * r, &sn, &cs);
            s.base[i * kBaseStride + gb] = make_float2(cs, sn);
        }
        __syncthreads();
        for (int q = 0; q < kTile / kSlices; ++q) {
            const int i = sl + kSlices * q;
            const float x = s.x32[i];
            const float r = fmaf(af, x, -rintf(af * x));
            float sa, ca;
            __sincosf(B2D_TWO_PI_F * r, &sa, &ca);
            const float us = s.u[i] * sa, uc = s.u[i] * ca;
            const float2* bs = s.base + i * kBaseStride;
#pragma unroll
            for (int gb = 0; gb < NBASE; ++gb) {
                const float2 cb = bs[gb];
                acc[gb] = fmaf(us, cb.x, fmaf(uc, cb.y, acc[gb]));   // u sin((hb + a) phi)
            }
        }
        __syncthreads();
    }
    // fixed-order reduction over the 8 sample slices; harmonic hh = 128 g + 16 b + a
    float* red = reinterpret_cast<float*>(s.base);     // [kSlices][128 G]
#pragma unroll
    for (int gb = 0; gb < NBASE; ++gb) red[sl * 128 * G + 128 * (gb >> 3) + 16 * (gb & 7) + a] = acc[gb];
    __syncthreads();
    const size_t fr = (size_t)b * nF + k;
    const float* crow = p.c_amp + fr * (size_t)p.ctrl_stride;
    const float f0k = p.f0[fr];
    float* grow = p.grad + fr * (size_t)p.grad_stride;
    for (int hh = tid; hh < p.H; hh += kThreads) {
        float dA = 0.f;
        for (int q = 0; q < kSlices; ++q) dA += red[q * 128 * G + hh];
        grow[hh] = dA * b2d_bank::activate_amp(crow[hh], f0k, hh, p.nyquist);
    }
}

}  // namespace

#ifndef B2D_HOST_EMU
namespace {
template <int G>
int bank_bwd_launch(const BankBwdParams& p, int B, cudaStream_t st) {
    sins_bank_bwd_kernel<G><<<dim3((unsigned)p.nF, (unsigned)B), kThreads, sizeof(BankSmem), st>>>(p);
    return b2d::check_launch("sins_synth_backward: bank");
}
}  // namespace

extern "C" size_t b2d_sins_synth_backward_workspace_bytes(int B, int n_frames, int block) {
    if (B <= 0 || n_frames <= 0 || block <= 0) return 0;
    return 2 * b2d::align256((size_t)B * n_frames * block * 4);     // dL/dsinusoids | sinusoids rebuilt when not in the forward's
}

extern "C" int b2d_sins_synth_backward(const float* f0_frames, const double* frame_phase, const float* c_amp,
                                       const float* c_group_delay, const float* c_noise, int64_t ctrl_stride,
                                       const float* noise_in, uint64_t seed, int64_t utterance_offset,
                                       const void* forward_workspace, int forward_has_sinusoids,
                                       const float* grad_signal, const float* grad_harmonic, const float* grad_noise,
                                       int B, int n_frames, int block, int n_harmonics, int n_mag_allpass,
                                       int n_mag_noise, double sampling_rate, float* grad_ctrl, void* workspace,
                                       size_t workspace_bytes, void* stream) {
    if (!f0_frames || !frame_phase || !c_amp || !c_group_delay || !c_noise || !forward_workspace || !grad_ctrl || !workspace)
        return b2d::fail(B2D_ERR_NULL, "sins_synth_backward: null pointer");
    if (B <= 0 || n_frames <= 0 || block <= 0 || n_harmonics <= 0 || n_mag_allpass < 2 || n_mag_noise < 2 ||
        ctrl_stride < n_harmonics || ctrl_stride < n_mag_allpass || ctrl_stride < n_mag_noise)
        return b2d::fail(B2D_ERR_SHAPE, "sins_synth_backward: bad shape B=%d nF=%d block=%d H=%d Ma=%d Mn=%d stride=%lld",
                         B, n_frames, block, n_harmonics, n_mag_allpass, n_mag_noise, (long long)ctrl_stride);
    if (block != kP || n_mag_allpass > kMaxBins || n_mag_noise > kMaxBins || n_harmonics > 512 || B > 65535)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "sins_synth_backward: built for block %d, n_mag <= %d, H <= 512, B <= 65535 "
                         "(got block %d, n_mag %d / %d, H %d, B %d)", kP, kMaxBins, block, n_mag_allpass, n_mag_noise,
                         n_harmonics, B);
    const size_t need = b2d_sins_synth_backward_workspace_bytes(B, n_frames, block);
    if (workspace_bytes < need)
        return b2d::fail(B2D_ERR_WORKSPACE, "sins_synth_backward: workspace %zu < %zu bytes", workspace_bytes, need);
    if ((reinterpret_cast<uintptr_t>(workspace) & 255u) || (reinterpret_cast<uintptr_t>(forward_workspace) & 255u) ||
        (noise_in && !b2d::aligned16(noise_in)) || (reinterpret_cast<uintptr_t>(grad_ctrl) & 3u))
        return b2d::fail(B2D_ERR_ALIGN, "sins_synth_backward: workspaces must be 256-byte aligned, noise_in 16-byte aligned");

    // the forward's buffers precede its spectrum buffers, so the spectrum flag does not move them
    const b2d::SinsWorkspace fw = b2d::sins_workspace(B, n_frames, block, n_mag_allpass, n_mag_noise, false);
    const float* sinus = b2d::ws_at(forward_workspace, fw.sinus);
    float* dx = static_cast<float*>(workspace);
    cudaStream_t st = (cudaStream_t)stream;
    if (!forward_has_sinusoids) {     // the fused forward evaluates the bank inside its FIR kernel: rebuild the sinusoids
        float* rebuilt = b2d::ws_at(workspace, b2d::align256((size_t)B * n_frames * block * 4));
        const int rc = b2d_sins_bank(f0_frames, frame_phase, c_amp, ctrl_stride, B, n_frames, block, n_harmonics,
                                     sampling_rate, 1, rebuilt, stream);
        if (rc) return rc;
        sinus = rebuilt;
    }

    FirBwdParams fp;
    fp.sinus = sinus; fp.noise_in = noise_in; fp.seed = seed; fp.utt_off = utterance_offset;
    fp.ir_ap = b2d::ws_at(forward_workspace, fw.ir_ap); fp.ir_n = b2d::ws_at(forward_workspace, fw.ir_n);
    fp.c_gd = c_group_delay; fp.c_nm = c_noise; fp.ctrl_stride = ctrl_stride;
    fp.g = grad_signal; fp.g_harm = grad_harmonic; fp.g_noise = grad_noise;
    fp.nF = n_frames; fp.Ma = n_mag_allpass; fp.Mn = n_mag_noise; fp.H = n_harmonics;
    fp.dx = dx; fp.grad = grad_ctrl;
    sins_fir_bwd_kernel<<<dim3((unsigned)n_frames, (unsigned)B), kThreads, sizeof(FirSmem), st>>>(fp);
    int rc = b2d::check_launch("sins_synth_backward: fir");
    if (rc) return rc;

    BankBwdParams bp;
    bp.f0 = f0_frames; bp.frame_phase = frame_phase; bp.c_amp = c_amp; bp.ctrl_stride = ctrl_stride; bp.dx = dx;
    bp.nF = n_frames; bp.H = n_harmonics; bp.inv_sr = 1.0 / sampling_rate; bp.nyquist = (float)(sampling_rate / 2.0);
    bp.grad = grad_ctrl; bp.grad_stride = (long long)n_harmonics + n_mag_allpass + n_mag_noise;
    switch ((n_harmonics + 127) / 128) {
        case 1: return bank_bwd_launch<1>(bp, B, st);
        case 2: return bank_bwd_launch<2>(bp, B, st);
        case 3: return bank_bwd_launch<3>(bp, B, st);
        default: return bank_bwd_launch<4>(bp, B, st);
    }
}
#endif  // B2D_HOST_EMU
