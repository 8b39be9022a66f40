// Random-scale spectral loss of the DDSP training step (ddsp/loss.py:9-54, RSSLoss / SSSLoss; train.py:82 builds it
// with fft_min 256, fft_max 2048, n_scale 4) and its gradient with respect to the prediction.  Per scale n:
//
//   frames   x[b, f n + m], m < n, f < F = 1 + (T - n) / n        (hop n: frames do not overlap; center = False)
//   S        = |rfft(w x_frame)| / c + eps,  w = periodic Hann(n), c = sqrt(sum w^2), K = n / 2 + 1 bins
//   loss_n   = mean_b ||S_t - S_p||_F / ||S_t + S_p||_F + alpha mean |log S_t - log S_p|
//   loss     = sum_n loss_n / n_scale
//
// Any n in [256, 2047] (primes included) goes through Bluestein's chirp z-transform (bluestein.cuh) for all n bins: size
// M = 1024 / 2048 / 4096, the smallest >= 2n - 1, so the first FFT skips the zero upper half of u (n <= M / 2).
//
// One CTA (128 threads) owns one frame of one row and runs two transforms side by side: the prediction's frame and the
// target's (see transform_frames for why frames are not packed two to a transform).  Both signals go through the same
// arithmetic, fixed by the frame index and not by the grid, so equal rows give bit-equal spectra and an exactly zero
// loss, as in the reference.
//
// rss_fwd_kernel writes, per frame, sum D^2, sum A^2 and sum |log S_t - log S_p| (D = S_t - S_p, A = S_t + S_p) in
// float64 to a workspace; rss_finalize_kernel (one CTA) reduces them in a fixed order to the per-(scale, row) norms
// ||D||, ||A|| and the fp32 loss scalar.  No atomics, no host synchronisation, and nothing depends on the grid.
//
// rss_bwd_kernel recomputes both spectra (nothing is stored between forward and backward) and applies
//   g_S = s [ (1/B)(-[||D|| > 0] D / (||D|| ||A||) - ||D|| A / ||A||^3) - alpha sign(log S_t - log S_p) / (B K F S_p) ]
//   G[k] = g_S[k] X[k] / (c |X[k]|)  (0 where |X| = 0),   dx[m] = w[m] Re sum_{k<K} G[k] e^{+2 pi i k m / n}
// with s = dL/dloss / n_scale.  The adjoint is one more Bluestein transform per frame, of G zero-padded to n:
// sum_{k<K} G[k] e^{+2 pi i k m / n} = DFT_n(G)[(n - m) mod n], of which dx takes the real part.
// Frames do not overlap, so every sample has one owner per scale: the first scale stores (zeros past the last frame),
// later scales add, launched in stream order.
#ifndef B2D_HOST_EMU               // tests/emu/ runs the kernels' source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif
#include "bluestein.cuh"

using namespace b2d_fft;
using namespace b2d_bluestein;
using b2d_fft_smem::kThreads;
using b2d_fft_smem::padi;

namespace {

constexpr int kNMin = 256, kNMax = 2047, kMaxScales = 64;

// per-n table (bluestein.cuh's layout): [0] c = sqrt(sum w^2), then the window, the chirp and FFT_M(h) / M
__host__ __device__ __forceinline__ int bluestein_size(int n) { return b2d_bluestein::bluestein_size(n, n); }

template <int M> constexpr size_t smem_bytes() {
    return (size_t)2 * b2d_fft_smem::Plan<M>::kPad * sizeof(float2) +
           (size_t)(b2d_fft_smem::Plan<M>::kTw2 + b2d_fft_smem::Plan<M>::kTw3) * sizeof(float2) +
           (size_t)3 * kThreads * sizeof(float);
}

struct RssParams {
    const float* xp;           // [B, T] prediction
    const float* xt;           // [B, T] target
    const float* table;        // per-n table (layout above)
    double* part;              // forward: [B, F, 3] per-frame sums of this scale
    const double* norms;       // backward: [B, 2] ||D||, ||A|| of this scale
    const float* grad_loss;    // backward: dL/dloss (device scalar)
    float* dx;                 // backward: [B, T]
    int T, n, F, B, accumulate;
    float alpha, eps;
    double inv_scales;         // 1 / n_scale
};

// shared-memory layout of both kernels: two padded M-point buffers, the twiddles, a [3][128] reduction area
template <int M> struct Smem {
    float2 *z0, *z1, *tw2, *tw3;
    float* red;
    __device__ __forceinline__ explicit Smem(unsigned char* raw) {
        z0 = reinterpret_cast<float2*>(raw);
        z1 = z0 + b2d_fft_smem::Plan<M>::kPad;
        tw2 = z1 + b2d_fft_smem::Plan<M>::kPad;
        tw3 = tw2 + b2d_fft_smem::Plan<M>::kTw2;
        red = reinterpret_cast<float*>(tw3 + b2d_fft_smem::Plan<M>::kTw3);
    }
};

// the windowed, chirped frame at x into z (w x conj(c) on [0, n)), zero on [n, M/2)
template <int M>
__device__ __forceinline__ void load_frame(float2* z, const float* __restrict__ x, const float* __restrict__ window,
                                           const float2* __restrict__ chirp, int n, int tid) {
    for (int m = tid; m < M / 2; m += kThreads) {
        float2 v = make_float2(0.f, 0.f);
        if (m < n) {
            const float a = __ldg(window + m) * __ldg(x + m);
            const float2 ch = __ldg(chirp + m);
            v = make_float2(a * ch.x, -a * ch.y);
        }
        z[padi(m)] = v;
    }
}

// S = |X / c| + eps; also the normalised spectrum and its magnitude (for the backward)
struct Bin { float xr, xi, mag, S; };
__device__ __forceinline__ Bin spec_bin(float2 X, float c, float eps) {
    Bin q;
    q.xr = X.x / c; q.xi = X.y / c;
    q.mag = sqrtf(q.xr * q.xr + q.xi * q.xi);
    q.S = q.mag + eps;
    return q;
}

// frame f of row b of both signals: load and transform (prediction in z0, target in z1); bin k of the prediction's
// spectrum is then bluestein_out(z0, k), the target's bluestein_out(z1, k).  One frame per transform: packing two
// frames as a + j b would leak round-off of order 2^-24 |b| into a through the conjugate-symmetric split, and a silent
// frame next to a loud one would get a spectrum far above eps instead of the reference's exact eps.
template <int M>
__device__ __forceinline__ void transform_frames(const Smem<M>& sm, const RssParams& p, int b, int f, int tid) {
    const float* tab = p.table;
    const float2* chirp = reinterpret_cast<const float2*>(tab + chirp_off(p.n));
    const float2* hspec = reinterpret_cast<const float2*>(tab + hspec_off(p.n));
    const size_t s0 = (size_t)b * p.T + (size_t)f * p.n;
    load_frame<M>(sm.z0, p.xp + s0, tab + kWinOff, chirp, p.n, tid);
    load_frame<M>(sm.z1, p.xt + s0, tab + kWinOff, chirp, p.n, tid);
    b2d_fft_smem::init_twiddles<M>(sm.tw2, sm.tw3, tid);
    __syncthreads();
    bluestein_core<M, 2>(sm.z0, hspec, sm.tw2, sm.tw3, tid);
}

template <int M>
__global__ void __launch_bounds__(kThreads) rss_fwd_kernel(RssParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const Smem<M> sm(smem_raw);
    const int tid = threadIdx.x, b = blockIdx.y, f = blockIdx.x;
    const float2* chirp = reinterpret_cast<const float2*>(p.table + chirp_off(p.n));
    const float c = __ldg(p.table);
    transform_frames<M>(sm, p, b, f, tid);
    // per-thread partial sums over bins k = tid, tid + 128, ... (fixed order)
    float d2 = 0.f, a2 = 0.f, l1 = 0.f;
    const int K = p.n / 2 + 1;
    for (int k = tid; k < K; k += kThreads) {
        const float sp = spec_bin(bluestein_out<M>(sm.z0, chirp, k), c, p.eps).S;
        const float st = spec_bin(bluestein_out<M>(sm.z1, chirp, k), c, p.eps).S;
        const float d = st - sp, a = st + sp;
        d2 = fmaf(d, d, d2); a2 = fmaf(a, a, a2); l1 += fabsf(logf(st) - logf(sp));
    }
    float* red = sm.red;
    red[0 * kThreads + tid] = d2; red[1 * kThreads + tid] = a2; red[2 * kThreads + tid] = l1;
    __syncthreads();
    if (tid < 3) {
        double s = 0.0;
        for (int i = 0; i < kThreads; ++i) s += (double)red[tid * kThreads + i];
        p.part[((size_t)b * p.F + f) * 3 + tid] = s;
    }
}

// One CTA: per (scale, row) norms in float64 (frames summed in order), then the loss in a fixed order.
struct RssFinalizeParams {
    const double* part;        // scale s at part + off[s]: [B, F[s], 3]
    double* norms;             // [n_scale, B, 2]
    float* loss;               // device scalar
    long long off[kMaxScales];
    int F[kMaxScales], K[kMaxScales];
    int B, n_scale;
    float alpha;
};

__global__ void __launch_bounds__(kThreads) rss_finalize_kernel(RssFinalizeParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double* red = reinterpret_cast<double*>(smem_raw);        // [2][128]
    const int tid = threadIdx.x;
    double total = 0.0;
    for (int s = 0; s < p.n_scale; ++s) {
        double conv = 0.0, l1 = 0.0;
        for (int b = tid; b < p.B; b += kThreads) {
            const double* q = p.part + p.off[s] + (size_t)b * p.F[s] * 3;
            double d2 = 0.0, a2 = 0.0, l = 0.0;
            for (int f = 0; f < p.F[s]; ++f) { d2 += q[3 * f]; a2 += q[3 * f + 1]; l += q[3 * f + 2]; }
            const double nd = sqrt(d2), na = sqrt(a2);
            p.norms[((size_t)s * p.B + b) * 2] = nd;
            p.norms[((size_t)s * p.B + b) * 2 + 1] = na;
            conv += nd / na;
            l1 += l;
        }
        red[tid] = conv; red[kThreads + tid] = l1;
        __syncthreads();
        if (tid == 0) {
            double c = 0.0, l = 0.0;
            for (int i = 0; i < kThreads; ++i) { c += red[i]; l += red[kThreads + i]; }
            total += c / p.B + (double)p.alpha * l / ((double)p.B * p.K[s] * p.F[s]);
        }
        __syncthreads();
    }
    if (tid == 0) p.loss[0] = (float)(total / p.n_scale);
}

template <int M>
__global__ void __launch_bounds__(kThreads) rss_bwd_kernel(RssParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const Smem<M> sm(smem_raw);
    const int tid = threadIdx.x, b = blockIdx.y, f = blockIdx.x, n = p.n;
    const float* window = p.table + kWinOff;
    const float2* chirp = reinterpret_cast<const float2*>(p.table + chirp_off(n));
    const float c = __ldg(p.table);
    const int K = n / 2 + 1;
    float* dx = p.dx + (size_t)b * p.T;
    if (!p.accumulate && blockIdx.x == 0)                     // the first scale owns the samples past its last frame
        for (int i = p.F * n + tid; i < p.T; i += kThreads) dx[i] = 0.f;
    // g_S = -c1 D - c2 A - c3 sign(log S_t - log S_p) / S_p   (torch: norm backward is 0 where the norm is 0)
    const double nd = p.norms[2 * b], na = p.norms[2 * b + 1];
    const double sc = (double)__ldg(p.grad_loss) * p.inv_scales;
    const float c1 = nd > 0.0 ? (float)(sc / (p.B * nd * na)) : 0.f;
    const float c2 = (float)(sc * nd / (p.B * na * na * na));
    const float c3 = (float)(sc * p.alpha / ((double)p.B * K * p.F));
    transform_frames<M>(sm, p, b, f, tid);
    // G[k], chirped, written in place into z0 slots [0, K), zeros on [K, M/2).  The transforms are read at slot 0 (by
    // bin 0's thread only, before it writes) and in (M - n, M), so no write lands on a slot another thread still reads.
    for (int k = tid; k < K; k += kThreads) {
        const Bin sp = spec_bin(bluestein_out<M>(sm.z0, chirp, k), c, p.eps);
        const Bin st = spec_bin(bluestein_out<M>(sm.z1, chirp, k), c, p.eps);
        const float lt = logf(st.S), lp = logf(sp.S);
        const float sgn = lt > lp ? 1.f : lt < lp ? -1.f : 0.f;
        const float gs = -c1 * (st.S - sp.S) - c2 * (st.S + sp.S) - c3 * sgn / sp.S;
        const float g = sp.mag > 0.f ? gs / (sp.mag * c) : 0.f;
        const float gr = g * sp.xr, gi = g * sp.xi;
        const float2 ck = __ldg(chirp + k);
        sm.z0[padi(k)] = make_float2(fmaf(gr, ck.x, gi * ck.y), fmaf(gi, ck.x, -gr * ck.y));      // G conj(c)
    }
    for (int m = K + tid; m < M / 2; m += kThreads) sm.z0[padi(m)] = make_float2(0.f, 0.f);
    __syncthreads();
    bluestein_core<M, 1>(sm.z0, reinterpret_cast<const float2*>(p.table + hspec_off(n)), sm.tw2, sm.tw3, tid);
    // sum_{k<K} G[k] e^{+2 pi i k m / n} = DFT_n(G zero-padded)[(n - m) mod n]; its real part is d[m]
    float* out = dx + (size_t)f * n;
    for (int m = tid; m < n; m += kThreads) {
        const float v = __ldg(window + m) * bluestein_out<M>(sm.z0, chirp, m == 0 ? 0 : n - m).x;
        out[m] = p.accumulate ? out[m] + v : v;
    }
}

}  // namespace

extern "C" int b2d_rss_table_floats(int n) {
    if (n < kNMin || n > kNMax) return 0;
    return bluestein_table_floats(n, n);
}

extern "C" int b2d_rss_frames(int n_samples, int n) {
    if (n < kNMin || n > kNMax || n_samples < n) return 0;
    return 1 + (n_samples - n) / n;
}

#ifndef B2D_HOST_EMU

namespace {

int check_args(const char* what, const float* xp, const float* xt, int B, int T, int n_scale, const int* n_ffts,
               const float* const* tables) {
    if (!xp || !xt || !n_ffts || !tables) return b2d::fail(B2D_ERR_NULL, "%s: null pointer", what);
    if (((uintptr_t)xp | (uintptr_t)xt) & 3) return b2d::fail(B2D_ERR_ALIGN, "%s: signals must be 4-byte aligned", what);
    if (B <= 0 || B > 65535 || T <= 0 || n_scale <= 0 || n_scale > kMaxScales)
        return b2d::fail(B2D_ERR_SHAPE, "%s: bad shape B=%d T=%d n_scale=%d (B <= 65535, n_scale <= %d)", what, B, T,
                         n_scale, kMaxScales);
    for (int s = 0; s < n_scale; ++s) {
        const int n = n_ffts[s];
        if (n < kNMin || n > kNMax)
            return b2d::fail(B2D_ERR_UNSUPPORTED, "%s: n_fft %d outside [%d, %d]", what, n, kNMin, kNMax);
        if (T < n) return b2d::fail(B2D_ERR_SHAPE, "%s: %d samples are shorter than n_fft %d", what, T, n);
        if (!tables[s]) return b2d::fail(B2D_ERR_NULL, "%s: null table for scale %d", what, s);
        if ((uintptr_t)tables[s] & 7) return b2d::fail(B2D_ERR_ALIGN, "%s: table of scale %d not 8-byte aligned", what, s);
    }
    return 0;
}

size_t part_doubles(int B, int T, int n) { return (size_t)B * b2d_rss_frames(T, n) * 3; }

template <int M> int launch_fwd(const RssParams& p, cudaStream_t st) {
    constexpr size_t smem = smem_bytes<M>();
    cudaError_t e = cudaFuncSetAttribute(rss_fwd_kernel<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return b2d::fail((int)e, "rss_loss_forward: smem attr: %s", cudaGetErrorString(e));
    rss_fwd_kernel<M><<<dim3(p.F, p.B), kThreads, smem, st>>>(p);
    return b2d::check_launch("rss_loss_forward");
}

template <int M> int launch_bwd(const RssParams& p, cudaStream_t st) {
    constexpr size_t smem = smem_bytes<M>();
    cudaError_t e = cudaFuncSetAttribute(rss_bwd_kernel<M>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return b2d::fail((int)e, "rss_loss_backward: smem attr: %s", cudaGetErrorString(e));
    rss_bwd_kernel<M><<<dim3(p.F, p.B), kThreads, smem, st>>>(p);
    return b2d::check_launch("rss_loss_backward");
}

}  // namespace

extern "C" size_t b2d_rss_loss_workspace_bytes(int B, int n_samples, int n_scale, const int* n_ffts) {
    if (!n_ffts || B <= 0 || n_scale <= 0 || n_scale > kMaxScales) return 0;
    size_t d = 0;
    for (int s = 0; s < n_scale; ++s) {
        if (b2d_rss_frames(n_samples, n_ffts[s]) <= 0) return 0;
        d += part_doubles(B, n_samples, n_ffts[s]);
    }
    return d * sizeof(double);
}

extern "C" int b2d_rss_loss_forward(const float* x_pred, const float* x_true, int B, int n_samples, int n_scale,
                                    const int* n_ffts, const float* const* tables, float alpha, float eps,
                                    void* workspace, size_t workspace_bytes, double* norms, float* loss, void* stream) {
    if (int rc = check_args("rss_loss_forward", x_pred, x_true, B, n_samples, n_scale, n_ffts, tables)) return rc;
    if (!workspace || !norms || !loss) return b2d::fail(B2D_ERR_NULL, "rss_loss_forward: null pointer");
    if (((uintptr_t)workspace | (uintptr_t)norms) & 7 || (uintptr_t)loss & 3)
        return b2d::fail(B2D_ERR_ALIGN, "rss_loss_forward: workspace / norms must be 8-byte aligned");
    if (workspace_bytes < b2d_rss_loss_workspace_bytes(B, n_samples, n_scale, n_ffts))
        return b2d::fail(B2D_ERR_WORKSPACE, "rss_loss_forward: workspace of %zu bytes is too small", workspace_bytes);
    cudaStream_t st = (cudaStream_t)stream;
    RssFinalizeParams fp;
    fp.part = (const double*)workspace; fp.norms = norms; fp.loss = loss; fp.B = B; fp.n_scale = n_scale; fp.alpha = alpha;
    long long off = 0;
    for (int s = 0; s < n_scale; ++s) {
        RssParams p = {};
        p.xp = x_pred; p.xt = x_true; p.table = tables[s]; p.part = (double*)workspace + off;
        p.T = n_samples; p.n = n_ffts[s]; p.F = b2d_rss_frames(n_samples, p.n); p.B = B;
        p.alpha = alpha; p.eps = eps;
        fp.off[s] = off; fp.F[s] = p.F; fp.K[s] = p.n / 2 + 1;
        off += (long long)part_doubles(B, n_samples, p.n);
        const int M = bluestein_size(p.n);
        const int rc = M == 1024 ? launch_fwd<1024>(p, st) : M == 2048 ? launch_fwd<2048>(p, st) : launch_fwd<4096>(p, st);
        if (rc) return rc;
    }
    rss_finalize_kernel<<<1, kThreads, 2 * kThreads * sizeof(double), st>>>(fp);
    return b2d::check_launch("rss_loss_finalize");
}

extern "C" int b2d_rss_loss_backward(const float* x_pred, const float* x_true, int B, int n_samples, int n_scale,
                                     const int* n_ffts, const float* const* tables, float alpha, float eps,
                                     const double* norms, const float* grad_loss, float* grad_pred, void* stream) {
    if (int rc = check_args("rss_loss_backward", x_pred, x_true, B, n_samples, n_scale, n_ffts, tables)) return rc;
    if (!norms || !grad_loss || !grad_pred) return b2d::fail(B2D_ERR_NULL, "rss_loss_backward: null pointer");
    if ((uintptr_t)norms & 7 || ((uintptr_t)grad_loss | (uintptr_t)grad_pred) & 3)
        return b2d::fail(B2D_ERR_ALIGN, "rss_loss_backward: norms must be 8-byte, grad_loss / grad_pred 4-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    for (int s = 0; s < n_scale; ++s) {
        RssParams p = {};
        p.xp = x_pred; p.xt = x_true; p.table = tables[s]; p.norms = norms + (size_t)s * B * 2; p.grad_loss = grad_loss;
        p.dx = grad_pred; p.T = n_samples; p.n = n_ffts[s]; p.F = b2d_rss_frames(n_samples, p.n); p.B = B;
        p.accumulate = s > 0; p.alpha = alpha; p.eps = eps; p.inv_scales = 1.0 / n_scale;
        const int M = bluestein_size(p.n);
        const int rc = M == 1024 ? launch_bwd<1024>(p, st) : M == 2048 ? launch_bwd<2048>(p, st) : launch_bwd<4096>(p, st);
        if (rc) return rc;
    }
    return 0;
}
#endif  // B2D_HOST_EMU
