// Direct-form adjoint of the time-varying FIR (ddsp/core.py:120-182) followed by the adjoint of the impulse-response
// build (ddsp/core.py:240-270), for one filter of one (frame, utterance) CTA: fir_adjoint, which serves the Sins
// backward (sins_bwd.cu: all-pass, noise) and the CombSub backward (combsub_bwd.cu: harmonic, noise; all-pass).  Every
// sum is a fixed-order fp32 / fp64 sum owned by one thread (block_scan: by one CTA), so no atomics.
#pragma once

namespace b2d_firadj {

constexpr int kP = 512;        // block size the backwards are built for
constexpr int kThreads = 128;  // one CTA per (frame, utterance); a thread owns 4 samples of a hop
constexpr int kSub = 16;       // irfft adjoint: n = kSub a + r, exact table twiddles per (bin, r) and per a

// inclusive prefix (reverse = false) or suffix (reverse = true) sums of val[0, n) in fp64 into out, for a CTA of NT
// threads.  Thread t owns scan positions [t per, (t + 1) per); the chunk totals are combined by a
// Hillis-Steele scan in part[2 NT].  The summation order depends only on n.  Ends with a barrier.
template <int NT>
__device__ void block_scan(const float* val, double* out, int n, bool reverse, double* part) {
    const int tid = threadIdx.x;
    const int per = (n + NT - 1) / NT;
    double run = 0.0;
    for (int q = 0; q < per; ++q) {
        const int pos = tid * per + q;
        if (pos < n) {
            const int i = reverse ? n - 1 - pos : pos;
            run += (double)val[i];
            out[i] = run;
        }
    }
    part[tid] = run;
    __syncthreads();
    int src = 0;
    for (int off = 1; off < NT; off <<= 1) {
        double s = part[src * NT + tid];
        if (tid >= off) s += part[src * NT + tid - off];
        part[(1 - src) * NT + tid] = s;
        __syncthreads();
        src = 1 - src;
    }
    const double before = tid > 0 ? part[src * NT + tid - 1] : 0.0;
    for (int q = 0; q < per; ++q) {
        const int pos = tid * per + q;
        if (pos < n) out[reverse ? n - 1 - pos : pos] += before;
    }
    __syncthreads();
}

// Filter-gradient correlation of four taps 4 t4 .. 4 t4 + 3 (shared memory, 16-byte aligned):
//   acc[k] += sum_{i < 4 nq} v[i] g[4 t4 + k + i]
// with an 8-float register window sliding along g (one float4 of g and one of v per 16 FMAs).
__device__ __forceinline__ void corr4(const float* g, const float* v, int t4, int nq, float acc[4]) {
    const float4* g4 = reinterpret_cast<const float4*>(g);
    const float4* v4 = reinterpret_cast<const float4*>(v);
    float4 cur = g4[t4];
    for (int q = 0; q < nq; ++q) {
        const float4 nx = g4[q + t4 + 1];
        const float4 vv = v4[q];
        const float w[8] = {cur.x, cur.y, cur.z, cur.w, nx.x, nx.y, nx.z, nx.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            acc[k] = fmaf(vv.x, w[k], acc[k]);
            acc[k] = fmaf(vv.y, w[k + 1], acc[k]);
            acc[k] = fmaf(vv.z, w[k + 2], acc[k]);
            acc[k] = fmaf(vv.w, w[k + 3], acc[k]);
        }
        cur = nx;
    }
}

// Input-gradient pass of four samples 4 t4 .. 4 t4 + 3 through two filters hA, hB of 4 L4 taps (zero-padded):
//   a[k] += sum_tau hA[tau] g[4 t4 + k + tau],  c[k] += sum_tau hB[tau] g[4 t4 + k + tau]
__device__ __forceinline__ void fir_t4(const float* g, const float* hA, const float* hB, int t4, int L4, float a[4],
                                       float c[4]) {
    const float4* g4 = reinterpret_cast<const float4*>(g);
    const float4* hA4 = reinterpret_cast<const float4*>(hA);
    const float4* hB4 = reinterpret_cast<const float4*>(hB);
    float4 cur = g4[t4];
    for (int u = 0; u < L4; ++u) {
        const float4 nx = g4[t4 + u + 1];
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
}

// Adjoint of torch's c2r irfft (n = N = 2 (M - 1)) at bin j < M, from the un-rolled impulse-response gradient dr:
//   C_j = sum_n dr[n] cos(2 pi j n / N),  S_j = sum_n dr[n] sin(2 pi j n / N),
// with eo[n] = (dr[n] + dr[N-n], dr[n] - dr[N-n]) for 1 <= n < N/2 (zero up to kSub nblk), d0 = dr[0], dN = dr[N/2],
// cosT / sinT = cos / sin(2 pi t / N).  n = kSub a + r: cos / sin of (alpha_a + beta_r) from the exact table entries of
// alpha_a and beta_r.  Returns dH_j = (dre, dim): weight 2/N, and 1/N with the imaginary part dropped at DC and Nyquist.
__device__ __forceinline__ void irfft_adjoint_bin(int j, int M, int N, int nblk, const float* cosT, const float* sinT,
                                                  const float2* eo, float d0, float dN, float& dre, float& dim) {
    float cb[kSub], sb[kSub];
#pragma unroll
    for (int r = 0; r < kSub; ++r) {
        const int idx = (j * r) % N;
        cb[r] = cosT[idx];
        sb[r] = sinT[idx];
    }
    float C = 0.f, S = 0.f;
    int ia = 0;
    const int step = (j * kSub) % N;
    for (int a = 0; a < nblk; ++a) {
        float U = 0.f, V = 0.f, U2 = 0.f, V2 = 0.f;
#pragma unroll
        for (int r = 0; r < kSub; ++r) {
            const float2 e = eo[a * kSub + r];
            U = fmaf(e.x, cb[r], U);
            V = fmaf(e.x, sb[r], V);
            U2 = fmaf(e.y, cb[r], U2);
            V2 = fmaf(e.y, sb[r], V2);
        }
        const float ca = cosT[ia], sa = sinT[ia];
        C = fmaf(ca, U, fmaf(-sa, V, C));          // sum e cos(alpha + beta)
        S = fmaf(sa, U2, fmaf(ca, V2, S));         // sum o sin(alpha + beta)
        ia += step;
        if (ia >= N) ia -= N;
    }
    C += d0 + ((j & 1) ? -dN : dN);
    const bool edge = (j == 0 || j == M - 1);
    const float wj = (edge ? 1.0f : 2.0f) / (float)N;
    dre = wj * C;
    dim = edge ? 0.f : -wj * S;
}

// The filter decides the window of the un-rolled impulse response and the activation of its raw control c:
//   kAllpass   no window; phi = cumsum(pi tanh c), dphi_j = Im(dH_j conj(H_j)), reverse cumsum, * pi (1 - tanh^2 c)
//   kHarmonic  the frame's dynamic raised cosine (ir_build_tc.cu's fp32 formula); Re(dH) exp(c)
//   kNoise     the periodic Hann window; Re(dH) exp(c) / 128
enum FirKind { kAllpass, kHarmonic, kNoise };

// One filter y = FIR(x, h) seen from the CTA of (frame f = blockIdx.x, utterance b = blockIdx.y); [B, T] rows, T = nF P
struct FirArgs {
    int nF, M;                // frames, bins (L = 2 (M - 1) taps)
    const float* x;           // filter input; kNoise: nullptr = in-kernel Philox noise keyed by (seed, utt_off + b)
    unsigned long long seed;
    long long utt_off;
    const float* g;           // cotangent g + g_add (nullptr = zero)
    const float* g_add;
    const float* ir;          // [B, nF, L] the forward's impulse responses, read when dx is set
    float* dx;                // [B, T] input gradient of hop f, or nullptr
    const float* f0;          // kHarmonic: this frame's f0, and 1.5 sr in fp32 (as ir_build.cu)
    float hw_num;
    const float* ctrl;        // this frame's raw control [M]
    float* grad_row;          // this frame's dense gradient row; the control's gradient starts at column col
    int col;
};

template <int kMaxTaps>
struct FirSmem {
    static constexpr int kWin = 2 * kP + kMaxTaps + 4;   // cotangent window (+ the register window's overhang)
    static constexpr int kMaxBins = kMaxTaps / 2 + 1;
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

// dh_f[tau] = sum_{i < 2P} v[i] g[(f-1)P + i - L/2 + tau], v = x weighted by phi (hop f-1) and 1 - phi (hop f; 1 at the
// last row, which also carries the held row nF); with dx, dx[fP + q] = (1 - phi) FIR^T(g, h_f) + phi FIR^T(g, h_{f+1});
// then un-roll dh, window, adjoint of torch's c2r irfft and the activation into grad_row.  A thread owns taps
// 4 t4 .. 4 t4 + 3 for t4 = tid, tid + 128, .. and samples 4 tid .. 4 tid + 3.  Restages every buffer; ends with a
// barrier.
template <FirKind kKind, int kMaxTaps>
__device__ __forceinline__ void fir_adjoint(FirSmem<kMaxTaps>& s, const FirArgs& p) {
    const int f = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const int nF = p.nF, M = p.M, L = 2 * (M - 1), N = L, half = L / 2;
    const long long T = (long long)nF * kP;
    const size_t row = (size_t)b * (size_t)T;
    const float* crow = p.ctrl;
    const long long n0 = (long long)(f - 1) * kP - half;

    // ---- stage: cotangent window, weighted input, filter rows, DFT table, raw activations ----
    for (int i = tid; i < FirSmem<kMaxTaps>::kWin; i += kThreads) {
        const long long n = n0 + i;
        float v = 0.f;
        if (i < 2 * kP + L - 1 && n >= 0 && n < T) {
            if (p.g) v = p.g[row + n];
            if (p.g_add) v += p.g_add[row + n];
        }
        s.gw[i] = v;
    }
    for (int q = tid; q < 2 * kP / 4; q += kThreads) {
        const int i = 4 * q;
        const long long m = (long long)(f - 1) * kP + i;
        float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
        if (m >= 0 && m < T) {          // whole quads: m and T are multiples of 4
            if (kKind != kNoise || p.x) x = *reinterpret_cast<const float4*>(p.x + row + m);
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
    if (p.dx) {
        const float* ir = p.ir + (size_t)b * nF * L;
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
    if (kKind == kAllpass)
        for (int j = tid; j < M; j += kThreads) s.tmp[j] = B2D_PI_F * tanhf(crow[j]);   // the forward's pi tanh(c)
    __syncthreads();

    // ---- dh: thread owns taps 4 t4 .. 4 t4 + 3 ----
#pragma unroll 1
    for (int grp = 0; grp < kMaxTaps / (4 * kThreads); ++grp) {
        const int t4 = tid + grp * kThreads;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        if (4 * t4 < L) corr4(s.gw, s.v, t4, 2 * kP / 4, acc);
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (4 * t4 + k < L) s.dh[4 * t4 + k] = acc[k];
    }
    // ---- input gradient of hop f: thread owns samples 4 tid .. 4 tid + 3 ----
    if (p.dx) {
        float a[4] = {0.f, 0.f, 0.f, 0.f}, c[4] = {0.f, 0.f, 0.f, 0.f};
        fir_t4(s.gw + kP, s.hA, s.hB, tid, (L + 3) / 4, a, c);
        float o[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float ph = (float)(4 * tid + k) * (1.0f / kP);
            o[k] = fmaf(1.0f - ph, a[k], ph * c[k]);
        }
        *reinterpret_cast<float4*>(p.dx + row + (size_t)f * kP + 4 * tid) = make_float4(o[0], o[1], o[2], o[3]);
    }
    if (kKind == kAllpass) block_scan<kThreads>(s.tmp, s.cum, M, false, s.part);   // forward phase phi_j (barrier)
    else __syncthreads();

    // ---- un-roll the causal form: dr[n] = dh[(n + L/2) mod L] times the window of that tap ----
    const float hw = kKind == kHarmonic ? p.hw_num / (*p.f0 + 1e-3f) : 1.f;
    auto dr = [&](int n) -> float {
        int t = n + half;
        if (t >= L) t -= L;
        const float v = s.dh[t];
        if (kKind == kAllpass) return v;
        if (kKind == kNoise) return v * (0.5f - 0.5f * s.cosT[t]);        // periodic Hann
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
        irfft_adjoint_bin(j, M, N, nblk, s.cosT, s.sinT, s.eo, s.d0, s.dN, dre, dim);
        if (kKind == kAllpass) {
            float sn, cs;
            sincosf((float)s.cum[j], &sn, &cs);
            s.tmp[j] = dim * cs - dre * sn;                    // dphi_j = Im(dH conj(H))
        } else if (kKind == kHarmonic) {
            p.grad_row[p.col + j] = dre * expf(crow[j]);
        } else {
            p.grad_row[p.col + j] = (dre * 0.0078125f) * expf(crow[j]);
        }
    }
    if (kKind == kAllpass) {
        __syncthreads();
        block_scan<kThreads>(s.tmp, s.cum, M, true, s.part);    // reverse cumsum: sum_{i >= j} dphi_i
        for (int j = tid; j < M; j += kThreads) {
            const float th = tanhf(crow[j]);
            p.grad_row[p.col + j] = ((float)s.cum[j] * B2D_PI_F) * (1.0f - th * th);
        }
    }
    __syncthreads();   // the next filter restages every buffer
}

}  // namespace b2d_firadj
