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

constexpr int kP = 512;                      // block size the backward is built for
constexpr int kMaxTaps = 512;                // 2 (n_mag - 1), n_mag <= 257
constexpr int kMaxBins = kMaxTaps / 2 + 1;
constexpr int kThreads = 128;
constexpr int kWin = 2 * kP + kMaxTaps + 4;  // cotangent window of one frame (+ the register window's overhang)
constexpr int kSub = 16;                     // DFT adjoint: n = kSub a + r, exact table twiddles per (bin, r) and per a

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

struct FirSmem {
    float gw[kWin];                    // cotangent window, origin at sample (f-1)P - L/2
    float v[2 * kP];                   // weighted filter input of hops f-1, f
    float hA[kMaxTaps], hB[kMaxTaps];  // h_f, h_{f+1}, zero-padded
    float dh[kMaxTaps];
    float cosT[kMaxTaps], sinT[kMaxTaps];   // cos / sin(2 pi t / N)
    float2 eo[kMaxTaps / 2];           // (dr[n] + dr[N-n], dr[n] - dr[N-n]) for 1 <= n < N/2, zero elsewhere
    float d0, dN;                      // dr[0], dr[N/2]
    float tmp[kMaxBins + 3];
    double cum[kMaxBins + 3];
    double part[2 * kThreads];
};

__global__ void __launch_bounds__(kThreads) sins_fir_bwd_kernel(FirBwdParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    FirSmem& s = *reinterpret_cast<FirSmem*>(smem_raw);
    const int f = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int nF = p.nF;
    const long long T = (long long)nF * kP;
    const size_t row = (size_t)b * (size_t)T;
    const size_t frow = (size_t)b * nF + f;
    float* grow = p.grad + frow * (size_t)(p.H + p.Ma + p.Mn);

    for (int branch = 0; branch < 2; ++branch) {
        const bool harm = branch == 0;
        const int M = harm ? p.Ma : p.Mn, L = 2 * (M - 1), N = L, half = L / 2;
        const float* ir = (harm ? p.ir_ap : p.ir_n) + (size_t)b * nF * L;
        const float* gadd = harm ? p.g_harm : p.g_noise;
        const float* crow = (harm ? p.c_gd : p.c_nm) + frow * (size_t)p.ctrl_stride;
        const long long n0 = (long long)(f - 1) * kP - half;

        // ---- stage: cotangent window, weighted input, filter rows, DFT table, raw activations ----
        for (int i = tid; i < kWin; i += kThreads) {
            const long long n = n0 + i;
            float v = 0.f;
            if (i < 2 * kP + L - 1 && n >= 0 && n < T) {
                if (p.g) v = p.g[row + n];
                if (gadd) v += gadd[row + n];
            }
            s.gw[i] = v;
        }
        for (int q = tid; q < 2 * kP / 4; q += kThreads) {
            const int i = 4 * q;
            const long long m = (long long)(f - 1) * kP + i;
            float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m >= 0 && m < T) {          // whole quads: m and T are multiples of 4
                if (harm) x = *reinterpret_cast<const float4*>(p.sinus + row + m);
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
        for (int j = tid; j < M; j += kThreads)
            s.tmp[j] = harm ? B2D_PI_F * tanhf(crow[j]) : 0.f;     // the forward's pi tanh(c), scanned below
        __syncthreads();

        // ---- dh: thread owns taps 4 tid .. 4 tid + 3; an 8-float register window slides along the cotangent ----
        {
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
            if (4 * tid < L) b2d_firadj::corr4(s.gw, s.v, tid, 2 * kP / 4, acc);
#pragma unroll
            for (int k = 0; k < 4; ++k)
                if (4 * tid + k < L) s.dh[4 * tid + k] = acc[k];
        }
        // ---- dx of hop f (all-pass filter only): thread owns samples 4 tid .. 4 tid + 3 ----
        if (harm) {
            float a[4] = {0.f, 0.f, 0.f, 0.f}, c[4] = {0.f, 0.f, 0.f, 0.f};
            const float4* g4 = reinterpret_cast<const float4*>(s.gw + kP);
            const float4* hA4 = reinterpret_cast<const float4*>(s.hA);
            const float4* hB4 = reinterpret_cast<const float4*>(s.hB);
            const int L4 = (L + 3) / 4;
            float4 cur = g4[tid];
            for (int u = 0; u < L4; ++u) {
                const float4 nx = g4[tid + u + 1];
                const float4 ha = hA4[u], hb = hB4[u];
                const float w[8] = {cur.x, cur.y, cur.z, cur.w, nx.x, nx.y, nx.z, nx.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    a[k] = fmaf(ha.x, w[k], a[k]);
                    a[k] = fmaf(ha.y, w[k + 1], a[k]);
                    a[k] = fmaf(ha.z, w[k + 2], a[k]);
                    a[k] = fmaf(ha.w, w[k + 3], a[k]);
                    c[k] = fmaf(hb.x, w[k], c[k]);
                    c[k] = fmaf(hb.y, w[k + 1], c[k]);
                    c[k] = fmaf(hb.z, w[k + 2], c[k]);
                    c[k] = fmaf(hb.w, w[k + 3], c[k]);
                }
                cur = nx;
            }
            float o[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float ph = (float)(4 * tid + k) * (1.0f / kP);
                o[k] = fmaf(1.0f - ph, a[k], ph * c[k]);
            }
            *reinterpret_cast<float4*>(p.dx + row + (size_t)f * kP + 4 * tid) = make_float4(o[0], o[1], o[2], o[3]);
        }
        if (harm) b2d_firadj::block_scan<kThreads>(s.tmp, s.cum, M, false, s.part);    // forward phase phi_j = cumsum(pi tanh c) (barrier)
        else __syncthreads();

        // ---- un-roll the causal form: dr[n] = dh[(n + L/2) mod L] (noise: times the Hann window of that tap) ----
        auto dr = [&](int n) -> float {
            int t = n + half;
            if (t >= L) t -= L;
            const float v = s.dh[t];
            return harm ? v : v * (0.5f - 0.5f * s.cosT[t]);
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

        // ---- adjoint of irfft per bin j:  C_j = sum_n dr[n] cos(2 pi j n / N),  S_j = sum_n dr[n] sin(2 pi j n / N);
        // n = kSub a + r: cos / sin of (alpha_a + beta_r) from the exact table entries of alpha_a and beta_r ----
        const int nblk = (half + kSub - 1) / kSub;
        for (int j = tid; j < M; j += kThreads) {
            float cb[kSub], sb[kSub];
#pragma unroll
            for (int r = 0; r < kSub; ++r) {
                const int idx = (j * r) % N;
                cb[r] = s.cosT[idx];
                sb[r] = s.sinT[idx];
            }
            float C = 0.f, S = 0.f;
            int ia = 0;
            const int step = (j * kSub) % N;
            for (int a = 0; a < nblk; ++a) {
                float U = 0.f, V = 0.f, U2 = 0.f, V2 = 0.f;
#pragma unroll
                for (int r = 0; r < kSub; ++r) {
                    const float2 e = s.eo[a * kSub + r];
                    U = fmaf(e.x, cb[r], U);
                    V = fmaf(e.x, sb[r], V);
                    U2 = fmaf(e.y, cb[r], U2);
                    V2 = fmaf(e.y, sb[r], V2);
                }
                const float ca = s.cosT[ia], sa = s.sinT[ia];
                C = fmaf(ca, U, fmaf(-sa, V, C));          // sum e cos(alpha + beta)
                S = fmaf(sa, U2, fmaf(ca, V2, S));         // sum o sin(alpha + beta)
                ia += step;
                if (ia >= N) ia -= N;
            }
            C += s.d0 + ((j & 1) ? -s.dN : s.dN);
            const bool edge = (j == 0 || j == M - 1);
            const float wj = (edge ? 1.0f : 2.0f) / (float)N;
            const float dre = wj * C, dim = edge ? 0.f : -wj * S;
            if (harm) {
                float sn, cs;
                sincosf((float)s.cum[j], &sn, &cs);
                s.tmp[j] = dim * cs - dre * sn;                // dphi_j = Im(dH conj(H))
            } else {
                const float c = crow[j];
                grow[p.H + p.Ma + j] = (dre * 0.0078125f) * expf(c);
            }
        }
        if (harm) {
            __syncthreads();
            b2d_firadj::block_scan<kThreads>(s.tmp, s.cum, M, true, s.part);          // reverse cumsum: d(pi tanh c)_j = sum_{i >= j} dphi_i
            for (int j = tid; j < M; j += kThreads) {
                const float th = tanhf(crow[j]);
                grow[p.H + j] = ((float)s.cum[j] * B2D_PI_F) * (1.0f - th * th);
            }
        }
        __syncthreads();   // the next branch restages every buffer
    }
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
inline size_t align256(size_t v) { return (v + 255) / 256 * 256; }

template <int G>
int bank_bwd_launch(const BankBwdParams& p, int B, cudaStream_t st) {
    sins_bank_bwd_kernel<G><<<dim3((unsigned)p.nF, (unsigned)B), kThreads, sizeof(BankSmem), st>>>(p);
    return b2d::check_launch("sins_synth_backward: bank");
}
}  // namespace

extern "C" size_t b2d_sins_synth_backward_workspace_bytes(int B, int n_frames, int block) {
    if (B <= 0 || n_frames <= 0 || block <= 0) return 0;
    return 2 * align256((size_t)B * n_frames * block * 4);     // dL/dsinusoids | sinusoids rebuilt when not in the forward's
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

    const size_t BT = (size_t)B * n_frames * block, BF = (size_t)B * n_frames;
    const int La = 2 * (n_mag_allpass - 1);
    const char* fws = static_cast<const char*>(forward_workspace);
    const float* ir_ap = reinterpret_cast<const float*>(fws + align256(BT * 4));
    const float* ir_n = reinterpret_cast<const float*>(fws + align256(BT * 4) + align256(BF * La * 4));
    char* ws = static_cast<char*>(workspace);
    float* dx = reinterpret_cast<float*>(ws);
    const float* sinus = reinterpret_cast<const float*>(fws);
    cudaStream_t st = (cudaStream_t)stream;
    if (!forward_has_sinusoids) {     // the fused forward evaluates the bank inside its FIR kernel: rebuild the sinusoids
        float* rebuilt = reinterpret_cast<float*>(ws + align256(BT * 4));
        const int rc = b2d_sins_bank(f0_frames, frame_phase, c_amp, ctrl_stride, B, n_frames, block, n_harmonics,
                                     sampling_rate, 1, rebuilt, stream);
        if (rc) return rc;
        sinus = rebuilt;
    }

    FirBwdParams fp;
    fp.sinus = sinus; fp.noise_in = noise_in; fp.seed = seed; fp.utt_off = utterance_offset;
    fp.ir_ap = ir_ap; fp.ir_n = ir_n; fp.c_gd = c_group_delay; fp.c_nm = c_noise; fp.ctrl_stride = ctrl_stride;
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
