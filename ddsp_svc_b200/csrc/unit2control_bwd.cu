// Backward of the fused frame-rate kernels of the control network with the convolution-only decoder (Unit2Control with
// use_naive_v2: ddsp/unit2control.py:84-109 + diffusion/model_conformer_naive.py): the adjoint of everything in
// unit2control.cu that the naive decoder runs.  The GEMM adjoints (dX = gY W, dW = gY^T X) are library GEMMs issued by
// the host side (ddsp_svc_b200/unit2control.py); these kernels sit between them:
//
//   u2c_glu_bwd        adjoint of GLU -> depthwise conv (k = 31) -> SiLU, recomputing the stage from the saved pw1 output
//   u2c_ln_bwd         LayerNorm: gx per token + per-slab column sums for dgamma / dbeta
//   u2c_gn_bwd_*       GroupNorm + LeakyReLU from the saved pre-norm activation and the forward's fp64 statistics
//   u2c_embed_bwd_*    gradient of the packed [7][256] embedding table + per-utterance row sums (speaker embedding)
//   u2c_colsum         column sum of a [N, O] cotangent: the bias gradient of every GEMM
//   u2c_conv3_fold     adjoint of the "three shifted inputs" gather of the k = 3 convolutions
//
// No atomics: every output element has one owner that sums in a fixed order.  Sums over tokens are two-stage: each CTA
// owns a FIXED slab of tokens (the slab size is a constant, not a function of the grid) and writes its partial sums to
// the caller's workspace; a second kernel adds the slabs in slab order in fp64.  So gradients are bit-identical from run
// to run and do not depend on the device's SM count.
#ifndef B2D_HOST_EMU               // tests/emu/ runs the GLU kernel's source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif

namespace {

constexpr int kC = 256;                          // model width of Unit2Control
constexpr int kDwK = 31, kDwHalf = 15, kDwTile = 64;
constexpr int kURows = kDwTile + 4 * kDwHalf;    // u = GLU output: the tile with a halo of 30 frames
constexpr int kGRows = kDwTile + 2 * kDwHalf;    // c / gc: the tile with a halo of 15 frames
constexpr int kGluSmemBytes = (kURows + kGRows) * 128 * (int)sizeof(float);
constexpr int kDwbStride = 32;                   // per channel: 31 tap gradients, then the bias gradient

__device__ __forceinline__ float u2c_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

// With u = value sigmoid(gate), c[t] = bias + sum_k w[k] u[t + k - 15], out = c sigmoid(c):
//   gc = gout sigmoid(c) (1 + c (1 - sigmoid(c)));  gu[t] = sum_k w[k] gc[t - k + 15]  (zero outside [0, T))
//   g_value = gu sigmoid(gate);  g_gate = gu value sigmoid(gate) (1 - sigmoid(gate))
//   dw[k] = sum_t gc[t] u[t + k - 15];  dbias = sum_t gc[t]      (this CTA's frames only -> part)
// One CTA per (utterance, 128 channels, 64 frames), one thread per channel.  Each thread owns column threadIdx.x of both
// shared arrays (they are per-thread scratch that registers cannot index dynamically): no value crosses threads, so the
// kernel needs no barrier.  u and c are evaluated with the forward kernel's expressions.
__global__ void __launch_bounds__(128) u2c_glu_bwd_kernel(const float* __restrict__ h, const float* __restrict__ w,
                                                          const float* __restrict__ bias, const float* __restrict__ gout,
                                                          float* __restrict__ gh, float* __restrict__ part /* [B][n_tiles][Ci][32] */,
                                                          int T, int Ci, int n_tiles) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float (*us)[128] = reinterpret_cast<float (*)[128]>(smem_raw);
    float (*gs)[128] = us + kURows;
    const int tile = blockIdx.x % n_tiles, b = blockIdx.y, tx = threadIdx.x;
    const int c = (blockIdx.x / n_tiles) * 128 + tx, t0 = tile * kDwTile;
    const float* hb = h + (size_t)b * T * (2 * Ci);
    for (int r = 0; r < kURows; ++r) {
        const int t = t0 - 2 * kDwHalf + r;
        float u = 0.f;
        if (t >= 0 && t < T) {
            const float* row = hb + (size_t)t * (2 * Ci);
            u = row[c] * u2c_sigmoid(row[Ci + c]);
        }
        us[r][tx] = u;
    }
    float wk[kDwK];
#pragma unroll
    for (int k = 0; k < kDwK; ++k) wk[k] = w[(size_t)c * kDwK + k];
    const float bs = bias[c];
    for (int r = 0; r < kGRows; ++r) {
        const int t = t0 - kDwHalf + r;
        float g = 0.f;
        if (t >= 0 && t < T) {
            float acc = bs;
#pragma unroll
            for (int k = 0; k < kDwK; ++k) acc = fmaf(wk[k], us[r + k][tx], acc);
            const float s = u2c_sigmoid(acc);
            g = gout[((size_t)b * T + t) * Ci + c] * (s * (1.0f + acc * (1.0f - s)));
        }
        gs[r][tx] = g;
    }
    float dw[kDwK], db = 0.f;
#pragma unroll
    for (int k = 0; k < kDwK; ++k) dw[k] = 0.f;
    for (int i = 0; i < kDwTile; ++i) {
        const int t = t0 + i;
        if (t >= T) break;
        float gu = 0.f;
#pragma unroll
        for (int k = 0; k < kDwK; ++k) gu = fmaf(wk[k], gs[i + 2 * kDwHalf - k][tx], gu);
        const float gc = gs[i + kDwHalf][tx];
        db += gc;
#pragma unroll
        for (int k = 0; k < kDwK; ++k) dw[k] = fmaf(gc, us[i + kDwHalf + k][tx], dw[k]);
        const float* row = hb + (size_t)t * (2 * Ci);
        const float a = row[c], s = u2c_sigmoid(row[Ci + c]);
        float* o = gh + ((size_t)b * T + t) * (2 * Ci);
        o[c] = gu * s;
        o[Ci + c] = gu * a * (s * (1.0f - s));
    }
    float* p = part + (((size_t)b * n_tiles + tile) * Ci + c) * kDwbStride;
#pragma unroll
    for (int k = 0; k < kDwK; ++k) p[k] = dw[k];
    p[kDwK] = db;
}

}  // namespace

#ifndef B2D_HOST_EMU

namespace {

constexpr int kSlab = 128;       // tokens one CTA of a token reduction owns (fixed: the summation order must not follow the grid)
constexpr int kGnSlab = 64;      // frames of one utterance per CTA of the GroupNorm backward

inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// out[j] = sum over slabs s (in order, fp64) of part[s * stride + j], j < n: the second stage of every token reduction
__global__ void __launch_bounds__(256) u2c_reduce_partials_kernel(const float* __restrict__ part, int n_slabs, size_t stride, int n,
                                                                  float* __restrict__ out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    double s = 0.0;
    for (int i = 0; i < n_slabs; ++i) s += (double)part[(size_t)i * stride + j];
    out[j] = (float)s;
}

// part[slab][col] = sum of g[n][col] over the slab's tokens in token order
__global__ void __launch_bounds__(256) u2c_colsum_kernel(const float* __restrict__ g, int n_tokens, int n_cols, float* __restrict__ part) {
    const int col = blockIdx.x * 256 + threadIdx.x, n0 = blockIdx.y * kSlab;
    if (col >= n_cols) return;
    const int n1 = min(n0 + kSlab, n_tokens);
    float s = 0.f;
    for (int n = n0; n < n1; ++n) s += g[(size_t)n * n_cols + col];
    part[(size_t)blockIdx.y * n_cols + col] = s;
}

// LayerNorm(256) backward: one warp per token (mean / rstd / xhat evaluated as the forward does);
// gx = rstd (g - mean(g) - xhat mean(g xhat)) with g = gy gamma;  part[slab][0][c] = sum gy xhat, part[slab][1][c] = sum gy.
// Warp w of the CTA takes tokens slab * 128 + w + 8 j in order; the 8 warps' sums are added in warp order.
__global__ void __launch_bounds__(256) u2c_ln_bwd_kernel(const float* __restrict__ x, const float* __restrict__ gy,
                                                         const float* __restrict__ gamma, float eps, int n_tokens,
                                                         float* __restrict__ gx, float* __restrict__ part) {
    constexpr int per = kC / 32;
    __shared__ float red[8][2][kC];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float ga[per], dg[per], db[per];
#pragma unroll
    for (int i = 0; i < per; ++i) { ga[i] = gamma[lane + 32 * i]; dg[i] = 0.f; db[i] = 0.f; }
    const int n1 = min((int)(blockIdx.x + 1) * kSlab, n_tokens);
    for (int n = blockIdx.x * kSlab + warp; n < n1; n += 8) {
        const float* row = x + (size_t)n * kC;
        const float* grow = gy + (size_t)n * kC;
        float v[per], g[per], s = 0.f;
#pragma unroll
        for (int i = 0; i < per; ++i) { v[i] = row[lane + 32 * i]; s += v[i]; }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
        const float mean = s / (float)kC;
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < per; ++i) { const float d = v[i] - mean; q += d * d; }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) q += __shfl_xor_sync(0xffffffffu, q, d);
        const float rstd = rsqrtf(q / (float)kC + eps);
        float m1 = 0.f, m2 = 0.f;
#pragma unroll
        for (int i = 0; i < per; ++i) {
            const float go = grow[lane + 32 * i];
            v[i] = (v[i] - mean) * rstd;                 // xhat
            g[i] = go * ga[i];
            m1 += g[i]; m2 += g[i] * v[i];
            dg[i] += go * v[i]; db[i] += go;
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) { m1 += __shfl_xor_sync(0xffffffffu, m1, d); m2 += __shfl_xor_sync(0xffffffffu, m2, d); }
        m1 /= (float)kC; m2 /= (float)kC;
        float* out = gx + (size_t)n * kC;
#pragma unroll
        for (int i = 0; i < per; ++i) out[lane + 32 * i] = rstd * (g[i] - m1 - v[i] * m2);
    }
#pragma unroll
    for (int i = 0; i < per; ++i) { red[warp][0][lane + 32 * i] = dg[i]; red[warp][1][lane + 32 * i] = db[i]; }
    __syncthreads();
    const int c = threadIdx.x;
    float a = 0.f, bsum = 0.f;
#pragma unroll
    for (int wv = 0; wv < 8; ++wv) { a += red[wv][0][c]; bsum += red[wv][1][c]; }
    part[(size_t)blockIdx.x * 2 * kC + c] = a;
    part[(size_t)blockIdx.x * 2 * kC + kC + c] = bsum;
}

// ---- GroupNorm(G, 256) + LeakyReLU backward.  With xhat = (x - mean) rstd, v = xhat gamma + beta, y = lrelu(v):
//   gz = gy (v >= 0 ? 1 : slope);  dgamma = sum gz xhat;  dbeta = sum gz;  gxh = gz gamma;
//   gx = rstd (gxh - S1 / n - xhat S2 / n),  S1 = sum gxh, S2 = sum gxh xhat over the (utterance, group), n = T C / G
struct GnCoef { float mu, mu_lo, rstd; };
__device__ __forceinline__ GnCoef gn_coef(const double* __restrict__ stats, int b, int g, int G, double n, float eps) {
    const double m = stats[((size_t)b * G + g) * 2] / n, var = fmax(stats[((size_t)b * G + g) * 2 + 1] / n - m * m, 0.0);
    GnCoef k;
    k.rstd = (float)(1.0 / sqrt(var + (double)eps)); k.mu = (float)m; k.mu_lo = (float)(m - (double)k.mu);   // as u2c_gn_apply_kernel
    return k;
}
// pass 1: per (utterance, slab of 64 frames, channel) the fp64 sums of gz and gz xhat -> partd[b][slab][2][256]
__global__ void __launch_bounds__(256) u2c_gn_bwd_sums_kernel(const float* __restrict__ x, const float* __restrict__ gy,
                                                              const double* __restrict__ stats, const float* __restrict__ gamma,
                                                              const float* __restrict__ beta, float eps, float slope, int T, int G,
                                                              double* __restrict__ partd) {
    const int b = blockIdx.y, c = threadIdx.x, cpg = kC / G;
    const GnCoef k = gn_coef(stats, b, c / cpg, G, (double)cpg * (double)T, eps);
    const float ga = gamma[c], be = beta[c];
    const int t1 = min((int)(blockIdx.x + 1) * kGnSlab, T);
    double a = 0.0, q = 0.0;
    for (int t = blockIdx.x * kGnSlab; t < t1; ++t) {
        const size_t i = ((size_t)b * T + t) * kC + c;
        const float xh = ((x[i] - k.mu) - k.mu_lo) * k.rstd;
        const float gz = gy[i] * (xh * ga + be >= 0.f ? 1.0f : slope);
        a += (double)gz; q += (double)gz * (double)xh;
    }
    double* p = partd + ((size_t)b * gridDim.x + blockIdx.x) * 2 * kC;
    p[c] = a; p[kC + c] = q;
}
// pass 2: every CTA adds the utterance's slabs in order (a few per channel), forms S1 / S2 of the four groups and writes gx
// of its slab; the CTA of slab 0 also writes the utterance's dgamma / dbeta -> partf[b][2][256]
__global__ void __launch_bounds__(256) u2c_gn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ gy,
                                                               const double* __restrict__ stats, const float* __restrict__ gamma,
                                                               const float* __restrict__ beta, float eps, float slope, int T, int G,
                                                               const double* __restrict__ partd, float* __restrict__ gx,
                                                               float* __restrict__ partf) {
    __shared__ double sh[2][kC];
    const int b = blockIdx.y, c = threadIdx.x, cpg = kC / G, g = c / cpg;
    const double n = (double)cpg * (double)T;
    const GnCoef k = gn_coef(stats, b, g, G, n, eps);
    const float ga = gamma[c], be = beta[c];
    double a = 0.0, q = 0.0;
    for (int s = 0; s < (int)gridDim.x; ++s) {
        const double* p = partd + ((size_t)b * gridDim.x + s) * 2 * kC;
        a += p[c]; q += p[kC + c];
    }
    if (blockIdx.x == 0) { partf[(size_t)b * 2 * kC + c] = (float)q; partf[(size_t)b * 2 * kC + kC + c] = (float)a; }
    sh[0][c] = a * (double)ga; sh[1][c] = q * (double)ga;
    __syncthreads();
    double s1 = 0.0, s2 = 0.0;
    for (int i = 0; i < cpg; ++i) { s1 += sh[0][g * cpg + i]; s2 += sh[1][g * cpg + i]; }
    const float m1 = (float)(s1 / n), m2 = (float)(s2 / n);
    const int t1 = min((int)(blockIdx.x + 1) * kGnSlab, T);
    for (int t = blockIdx.x * kGnSlab; t < t1; ++t) {
        const size_t i = ((size_t)b * T + t) * kC + c;
        const float xh = ((x[i] - k.mu) - k.mu_lo) * k.rstd;
        const float gz = gy[i] * (xh * ga + be >= 0.f ? 1.0f : slope);
        gx[i] = k.rstd * (gz * ga - m1 - xh * m2);
    }
}

// ---- embedding sum backward: x += w_f0 lf + b_f0 + w_ph ph + b_ph + w_vol vol + b_vol + spk[b] + w_aug aug_b / 5 ----
// pass 1: part[b][slab][4][256] = sum over the slab's frames of g lf, g ph, g vol, g  (lf, ph as u2c_embed_kernel evaluates them)
__global__ void __launch_bounds__(256) u2c_embed_bwd_sums_kernel(const float* __restrict__ gx, const float* __restrict__ f0,
                                                                 const float* __restrict__ phase, const float* __restrict__ volume,
                                                                 int T, float* __restrict__ part) {
    const int b = blockIdx.y, c = threadIdx.x;
    const int t1 = min((int)(blockIdx.x + 1) * kSlab, T);
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
    for (int t = blockIdx.x * kSlab; t < t1; ++t) {
        const size_t n = (size_t)b * T + t;
        const float g = gx[n * kC + c];
        s0 = fmaf(g, logf(1.0f + __ldg(f0 + n) / 700.0f), s0);
        s1 = fmaf(g, __ldg(phase + n) / B2D_PI_F, s1);
        s2 = fmaf(g, __ldg(volume + n), s2);
        s3 += g;
    }
    float* p = part + ((size_t)b * gridDim.x + blockIdx.x) * 4 * kC;
    p[c] = s0; p[kC + c] = s1; p[2 * kC + c] = s2; p[3 * kC + c] = s3;
}
// pass 2 (one CTA, one thread per channel): utterances and slabs in order, fp64
__global__ void __launch_bounds__(256) u2c_embed_bwd_reduce_kernel(const float* __restrict__ part, const float* __restrict__ aug, int B,
                                                                   int n_slabs, float* __restrict__ dtable, float* __restrict__ rowsum) {
    const int c = threadIdx.x;
    double t0 = 0.0, t1 = 0.0, t2 = 0.0, tb = 0.0, ta = 0.0;
    for (int b = 0; b < B; ++b) {
        double rs = 0.0;
        for (int s = 0; s < n_slabs; ++s) {
            const float* p = part + ((size_t)b * n_slabs + s) * 4 * kC;
            t0 += (double)p[c]; t1 += (double)p[kC + c]; t2 += (double)p[2 * kC + c]; rs += (double)p[3 * kC + c];
        }
        rowsum[(size_t)b * kC + c] = (float)rs;
        tb += rs;
        if (aug) ta += rs * (double)(aug[b] / 5.0f);
    }
    dtable[c] = (float)t0; dtable[2 * kC + c] = (float)t1; dtable[4 * kC + c] = (float)t2;
    dtable[kC + c] = dtable[3 * kC + c] = dtable[5 * kC + c] = (float)tb;
    dtable[6 * kC + c] = (float)ta;
}

// cat[t] = (x[t-1], x[t], x[t+1]) with zero padding  =>  gx[t] = gcat[t+1][0:I] + gcat[t][I:2I] + gcat[t-1][2I:3I]
__global__ void __launch_bounds__(256) u2c_conv3_fold_kernel(const float* __restrict__ gcat, int T, int I, size_t total,
                                                             float* __restrict__ gx) {
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const size_t n = e / I;
        const int i = (int)(e - n * I), t = (int)(n % T);
        const float* row = gcat + n * 3 * I;
        float v = row[I + i];
        if (t + 1 < T) v += row[3 * I + i];
        if (t > 0) v += row[-3 * I + 2 * I + i];
        gx[e] = v;
    }
}

size_t glu_ws(int B, int T, int Ci) { return (size_t)B * cdiv(T, kDwTile) * Ci * kDwbStride * sizeof(float); }
size_t colsum_ws(int n_tokens, int n_cols) { return (size_t)cdiv(n_tokens, kSlab) * n_cols * sizeof(float); }
size_t gn_ws_d(int B, int T) { return b2d::align256((size_t)B * cdiv(T, kGnSlab) * 2 * kC * sizeof(double)); }
size_t gn_ws(int B, int T) { return gn_ws_d(B, T) + (size_t)B * 2 * kC * sizeof(float); }
size_t embed_ws(int B, int T) { return (size_t)B * cdiv(T, kSlab) * 4 * kC * sizeof(float); }

int reduce(const float* part, int n_slabs, size_t stride, int n, float* out, cudaStream_t st, const char* what) {
    u2c_reduce_partials_kernel<<<cdiv(n, 256), 256, 0, st>>>(part, n_slabs, stride, n, out);
    return b2d::check_launch(what);
}

}  // namespace

extern "C" size_t b2d_u2c_backward_workspace_bytes(int B, int T, int inner_channels, int max_cols) {
    if (B <= 0 || T <= 0 || inner_channels <= 0 || max_cols <= 0 || (long long)B * T > 0x7fffffffLL) return 0;
    size_t n = glu_ws(B, T, inner_channels);
    n = max(n, colsum_ws(B * T, max(max_cols, 2 * kC)));
    n = max(n, gn_ws(B, T));
    n = max(n, embed_ws(B, T));
    return b2d::align256(n);
}

extern "C" int b2d_u2c_glu_dwconv_silu_backward(const float* h, const float* weight, const float* bias, const float* gout, float* gh,
                                                float* dwb, int B, int T, int inner_channels, int kernel_size, void* ws,
                                                size_t ws_bytes, void* stream) {
    if (!h || !weight || !bias || !gout || !gh || !dwb || !ws) return b2d::fail(B2D_ERR_NULL, "u2c_glu_dwconv_silu_backward: null pointer");
    if (B <= 0 || T <= 0 || inner_channels <= 0 || inner_channels % 128 || kernel_size != kDwK || B > 65535)
        return b2d::fail(B2D_ERR_SHAPE, "u2c_glu_dwconv_silu_backward: needs kernel size 31 and channels multiple of 128");
    if (ws_bytes < glu_ws(B, T, inner_channels)) return b2d::fail(B2D_ERR_WORKSPACE, "u2c_glu_dwconv_silu_backward: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    static const cudaError_t attr = cudaFuncSetAttribute(u2c_glu_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kGluSmemBytes);
    if (attr != cudaSuccess) return b2d::fail((int)attr, "u2c_glu_dwconv_silu_backward: shared memory: %s", cudaGetErrorString(attr));
    const int n_tiles = cdiv(T, kDwTile);
    float* part = static_cast<float*>(ws);
    u2c_glu_bwd_kernel<<<dim3(n_tiles * (inner_channels / 128), B), 128, kGluSmemBytes, st>>>(h, weight, bias, gout, gh, part, T,
                                                                                             inner_channels, n_tiles);
    if (int rc = b2d::check_launch("u2c_glu_dwconv_silu_backward")) return rc;
    const int n = inner_channels * kDwbStride;
    return reduce(part, B * n_tiles, (size_t)n, n, dwb, st, "u2c_glu_dwconv_silu_backward: reduce");
}

extern "C" int b2d_u2c_colsum(const float* g, int n_tokens, int n_cols, float* out, void* ws, size_t ws_bytes, void* stream) {
    if (!g || !out || !ws) return b2d::fail(B2D_ERR_NULL, "u2c_colsum: null pointer");
    if (n_tokens <= 0 || n_cols <= 0 || cdiv(n_tokens, kSlab) > 65535) return b2d::fail(B2D_ERR_SHAPE, "u2c_colsum: bad shape");
    if (ws_bytes < colsum_ws(n_tokens, n_cols)) return b2d::fail(B2D_ERR_WORKSPACE, "u2c_colsum: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    float* part = static_cast<float*>(ws);
    const int n_slabs = cdiv(n_tokens, kSlab);
    u2c_colsum_kernel<<<dim3(cdiv(n_cols, 256), n_slabs), 256, 0, st>>>(g, n_tokens, n_cols, part);
    if (int rc = b2d::check_launch("u2c_colsum")) return rc;
    return reduce(part, n_slabs, (size_t)n_cols, n_cols, out, st, "u2c_colsum: reduce");
}

extern "C" int b2d_u2c_layernorm_backward(const float* x, const float* gy, const float* gamma, float eps, int n_tokens, int C,
                                          float* gx, float* dgamma_dbeta, void* ws, size_t ws_bytes, void* stream) {
    if (!x || !gy || !gamma || !gx || !dgamma_dbeta || !ws) return b2d::fail(B2D_ERR_NULL, "u2c_layernorm_backward: null pointer");
    if (n_tokens <= 0 || C != kC) return b2d::fail(B2D_ERR_SHAPE, "u2c_layernorm_backward: needs C = 256");
    if (ws_bytes < colsum_ws(n_tokens, 2 * kC)) return b2d::fail(B2D_ERR_WORKSPACE, "u2c_layernorm_backward: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    float* part = static_cast<float*>(ws);
    const int n_slabs = cdiv(n_tokens, kSlab);
    u2c_ln_bwd_kernel<<<n_slabs, 256, 0, st>>>(x, gy, gamma, eps, n_tokens, gx, part);
    if (int rc = b2d::check_launch("u2c_layernorm_backward")) return rc;
    return reduce(part, n_slabs, (size_t)2 * kC, 2 * kC, dgamma_dbeta, st, "u2c_layernorm_backward: reduce");
}

extern "C" int b2d_u2c_groupnorm_lrelu_backward(const float* x_pre, const double* stats, const float* gamma, const float* beta,
                                                float eps, float slope, const float* gy, int B, int T, int C, int groups, float* gx,
                                                float* dgamma_dbeta, void* ws, size_t ws_bytes, void* stream) {
    if (!x_pre || !stats || !gamma || !beta || !gy || !gx || !dgamma_dbeta || !ws)
        return b2d::fail(B2D_ERR_NULL, "u2c_groupnorm_lrelu_backward: null pointer");
    if (B <= 0 || T <= 0 || C != kC || groups <= 0 || C % groups || B > 65535)
        return b2d::fail(B2D_ERR_SHAPE, "u2c_groupnorm_lrelu_backward: needs C = 256");
    if (ws_bytes < gn_ws(B, T)) return b2d::fail(B2D_ERR_WORKSPACE, "u2c_groupnorm_lrelu_backward: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    double* partd = static_cast<double*>(ws);
    float* partf = reinterpret_cast<float*>(static_cast<char*>(ws) + gn_ws_d(B, T));
    const dim3 grid(cdiv(T, kGnSlab), B);
    u2c_gn_bwd_sums_kernel<<<grid, kC, 0, st>>>(x_pre, gy, stats, gamma, beta, eps, slope, T, groups, partd);
    u2c_gn_bwd_apply_kernel<<<grid, kC, 0, st>>>(x_pre, gy, stats, gamma, beta, eps, slope, T, groups, partd, gx, partf);
    if (int rc = b2d::check_launch("u2c_groupnorm_lrelu_backward")) return rc;
    return reduce(partf, B, (size_t)2 * kC, 2 * kC, dgamma_dbeta, st, "u2c_groupnorm_lrelu_backward: reduce");
}

extern "C" int b2d_u2c_embed_backward(const float* gx, const float* f0, const float* phase, const float* volume,
                                      const float* aug_shift, int B, int T, float* dtable, float* rowsum, void* ws, size_t ws_bytes,
                                      void* stream) {
    if (!gx || !f0 || !phase || !volume || !dtable || !rowsum || !ws) return b2d::fail(B2D_ERR_NULL, "u2c_embed_backward: null pointer");
    if (B <= 0 || T <= 0 || B > 65535) return b2d::fail(B2D_ERR_SHAPE, "u2c_embed_backward: bad shape");
    if (ws_bytes < embed_ws(B, T)) return b2d::fail(B2D_ERR_WORKSPACE, "u2c_embed_backward: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    float* part = static_cast<float*>(ws);
    const int n_slabs = cdiv(T, kSlab);
    u2c_embed_bwd_sums_kernel<<<dim3(n_slabs, B), kC, 0, st>>>(gx, f0, phase, volume, T, part);
    u2c_embed_bwd_reduce_kernel<<<1, kC, 0, st>>>(part, aug_shift, B, n_slabs, dtable, rowsum);
    return b2d::check_launch("u2c_embed_backward");
}

extern "C" int b2d_u2c_conv3_fold(const float* gcat, int B, int T, int channels, float* gx, void* stream) {
    if (!gcat || !gx) return b2d::fail(B2D_ERR_NULL, "u2c_conv3_fold: null pointer");
    if (B <= 0 || T <= 0 || channels <= 0) return b2d::fail(B2D_ERR_SHAPE, "u2c_conv3_fold: bad shape");
    const size_t total = (size_t)B * T * channels;
    const size_t blocks = min((total + 255) / 256, (size_t)b2d::num_sms() * 16);
    u2c_conv3_fold_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(gcat, T, channels, total, gx);
    return b2d::check_launch("u2c_conv3_fold");
}

#endif  // B2D_HOST_EMU
