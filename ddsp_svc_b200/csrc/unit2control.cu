// Fused frame-rate kernels of the control network (Unit2Control inference, SURVEY 8f rank 1): everything in
// ddsp/unit2control.py:84-109 + ddsp/pcmer.py / diffusion/model_conformer_naive.py that is NOT a plain GEMM.  The GEMMs
// (k = 3 convolutions as three shifted products, 1 x 1 convolutions, attention projections, dense_out) are library
// GEMMs issued by the host side (ddsp_svc_b200/unit2control.py); between them the activations [B, T, C] (token-major,
// C contiguous) pass through these kernels exactly once each:
//
//   u2c_embed           x += f0_embed(log(1 + f0/700)) + phase_embed(phase/pi) + volume_embed(volume) + spk (+ aug)  (:93-102)
//   u2c_groupnorm_lrelu GroupNorm(4, 256) over (64 channels x T) per utterance + LeakyReLU(0.01)                      (:50-52)
//   u2c_layernorm       LayerNorm(C) per token                                                (pcmer.py:143,209; :104)
//   u2c_glu_dwconv_silu GLU -> depthwise Conv1d(k = 31, same padding) -> SiLU                  (pcmer.py:211-215)
//   u2c_softmax_feat    performer softmax-kernel feature map of queries / keys after the projection GEMM (pcmer.py:13-48)
//
// All are HBM-bound elementwise / small-stencil passes: one read and one write of the activation, fp32 throughout.
#include "b2d_common.cuh"
#include "tf32_split.cuh"

namespace {

constexpr int kC = 256;     // model width of Unit2Control (fixed by the reference: every embed / norm is 256 wide)

// x [N, 256] += w_f0 * log(1 + f0/700) + b_f0 + w_ph * (phase/pi) + b_ph + w_vol * vol + b_vol + spk[b] (+ w_aug * aug/5)
__global__ void __launch_bounds__(256) u2c_embed_kernel(float* __restrict__ x, const float* __restrict__ f0,
                                                        const float* __restrict__ phase, const float* __restrict__ volume,
                                                        const float* __restrict__ emb /* [7][256]: wf bf wp bp wv bv wa */,
                                                        const float* __restrict__ spk /* [B or 1][256] or null */, int spk_rows,
                                                        const float* __restrict__ aug /* [B] or null */, int n_tokens, int T) {
    const int c = threadIdx.x;
    const float wf = emb[c], bf = emb[kC + c], wp = emb[2 * kC + c], bp = emb[3 * kC + c], wv = emb[4 * kC + c],
                bv = emb[5 * kC + c], wa = emb[6 * kC + c];
    for (int n = blockIdx.x; n < n_tokens; n += gridDim.x) {
        const int b = n / T;
        const float lf = logf(1.0f + __ldg(f0 + n) / 700.0f);
        const float ph = __ldg(phase + n) / B2D_PI_F;
        float v = x[(size_t)n * kC + c];
        v = v + (wf * lf + bf) + (wp * ph + bp) + (wv * __ldg(volume + n) + bv);        // the reference's association
        if (spk) v += spk[(size_t)(spk_rows == 1 ? 0 : b) * kC + c];
        if (aug) v += wa * (__ldg(aug + b) / 5.0f);
        x[(size_t)n * kC + c] = v;
    }
}

// ---- GroupNorm(G groups of C/G channels, statistics over channels x T of one utterance) + LeakyReLU, in place ----
// pass 1: partial sums per (b, g, slab of frames) in fp64 -> stats[b][g][2]   (atomics on doubles: order-insensitive enough,
//         the values feed a mean / variance that the reference itself accumulates in a different order)
__global__ void __launch_bounds__(256) u2c_gn_stats_kernel(const float* __restrict__ x, int T, int C, int G, double* __restrict__ stats) {
    const int b = blockIdx.y, cpg = C / G;
    const int c = threadIdx.x % C;                 // blockDim = C (256)
    const int g = c / cpg;
    double s = 0.0, ss = 0.0;
    for (int t = blockIdx.x; t < T; t += gridDim.x) {
        const float v = x[((size_t)b * T + t) * C + c];
        s += (double)v; ss += (double)v * (double)v;
    }
    // reduce over the cpg channels of the group inside the block (cpg = 64 = two warps)
    __shared__ double sh[2][256];
    sh[0][threadIdx.x] = s; sh[1][threadIdx.x] = ss;
    __syncthreads();
    if (c % cpg == 0) {
        double a = 0.0, q = 0.0;
        for (int i = 0; i < cpg; ++i) { a += sh[0][c + i]; q += sh[1][c + i]; }
        atomicAdd(stats + ((size_t)b * G + g) * 2, a);
        atomicAdd(stats + ((size_t)b * G + g) * 2 + 1, q);
    }
}
__global__ void __launch_bounds__(256) u2c_gn_apply_kernel(float* __restrict__ x, int T, int C, int G, const double* __restrict__ stats,
                                                           const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                           float slope) {
    const int b = blockIdx.y, cpg = C / G, c = threadIdx.x, g = c / cpg;
    const double n = (double)cpg * (double)T;
    const double mean = stats[((size_t)b * G + g) * 2] / n;
    const double var = fmax(stats[((size_t)b * G + g) * 2 + 1] / n - mean * mean, 0.0);
    // the mean as an unevaluated fp32 pair: rounding it to one float would shift a group whose mean is large against its
    // spread by up to half an ulp of the mean (mean / std = 1e3: 3e-5 std)
    const float rstd = (float)(1.0 / sqrt(var + (double)eps)), mu = (float)mean, mu_lo = (float)(mean - (double)mu);
    const float ga = gamma[c], be = beta[c];
    for (int t = blockIdx.x; t < T; t += gridDim.x) {
        const size_t i = ((size_t)b * T + t) * C + c;
        float v = ((x[i] - mu) - mu_lo) * rstd * ga + be;
        x[i] = v >= 0.f ? v : v * slope;
    }
}

// ---- LayerNorm over the last dimension (C <= 1024, multiple of 32), one warp per token ----
__global__ void __launch_bounds__(256) u2c_layernorm_kernel(const float* __restrict__ x, float* __restrict__ y, int n_tokens, int C,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta, float eps) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= n_tokens) return;
    const float* row = x + (size_t)warp * C;
    float v[32];
    const int per = C / 32;                         // <= 32
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) if (i < per) { v[i] = row[lane + 32 * i]; s += v[i]; }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    const float mean = s / (float)C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) if (i < per) { const float d = v[i] - mean; q += d * d; }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) q += __shfl_xor_sync(0xffffffffu, q, d);
    const float rstd = rsqrtf(q / (float)C + eps);
    float* out = y + (size_t)warp * C;
#pragma unroll
    for (int i = 0; i < 32; ++i) if (i < per) {
        const int c = lane + 32 * i;
        out[c] = (v[i] - mean) * rstd * gamma[c] + beta[c];
    }
}

// ---- GLU -> depthwise conv (k = 31, zero "same" padding 15 / 15) -> SiLU ----
// in [B, T, 2 Ci] (value channels 0..Ci-1, gate channels Ci..2Ci-1), w [Ci, 31], bias [Ci] -> out [B, T, Ci]
constexpr int kDwK = 31, kDwHalf = 15, kDwTile = 64;
__global__ void __launch_bounds__(128) u2c_glu_dwconv_silu_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                                  const float* __restrict__ bias, float* __restrict__ out, int T, int Ci) {
    __shared__ float tile[kDwTile + 2 * kDwHalf][128];
    const int b = blockIdx.z, c0 = blockIdx.y * 128, t0 = blockIdx.x * kDwTile, c = c0 + threadIdx.x;
    for (int r = 0; r < kDwTile + 2 * kDwHalf; ++r) {
        const int t = t0 - kDwHalf + r;
        float g = 0.f;
        if (t >= 0 && t < T) {
            const float* row = in + ((size_t)b * T + t) * (2 * Ci);
            const float a = row[c], gate = row[Ci + c];
            g = a * (1.0f / (1.0f + expf(-gate)));                      // out * gate.sigmoid()
        }
        tile[r][threadIdx.x] = g;
    }
    __syncthreads();
    float wk[kDwK];
#pragma unroll
    for (int k = 0; k < kDwK; ++k) wk[k] = w[(size_t)c * kDwK + k];
    const float bs = bias[c];
    for (int i = 0; i < kDwTile; ++i) {
        const int t = t0 + i;
        if (t >= T) break;
        float acc = bs;
#pragma unroll
        for (int k = 0; k < kDwK; ++k) acc = fmaf(wk[k], tile[i + k][threadIdx.x], acc);   // cross-correlation, like Conv1d
        out[((size_t)b * T + t) * Ci + c] = acc * (1.0f / (1.0f + expf(-acc)));            // SiLU
    }
}

// ---- performer softmax-kernel feature map (pcmer.py:13-48), in place on dd = (d^-1/4 data) proj^T  [rows, J] ----
//   query: ratio * (exp(dd - diag - max_j dd) + eps);  key: ratio * exp(dd - diag + eps);  diag = |data|^2 / 2 * d^-1/2
__global__ void __launch_bounds__(256) u2c_softmax_feat_kernel(float* __restrict__ dd, const float* __restrict__ data, int rows, int J,
                                                               int d, int is_query, float eps) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const float* x = data + (size_t)warp * d;
    float sq = 0.f;
    for (int i = lane; i < d; i += 32) { const float v = x[i]; sq += v * v; }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, s);
    const float normalizer = rsqrtf(sqrtf((float)d));                    // d ** -0.25
    const float diag = (sq / 2.0f) * (normalizer * normalizer);
    const float ratio = rsqrtf((float)J);
    float* r = dd + (size_t)warp * J;
    float mx = -INFINITY;
    if (is_query) {
        for (int j = lane; j < J; j += 32) mx = fmaxf(mx, r[j]);
#pragma unroll
        for (int s = 16; s > 0; s >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, s));
    }
    for (int j = lane; j < J; j += 32)
        r[j] = is_query ? ratio * (expf(r[j] - diag - mx) + eps) : ratio * expf(r[j] - diag + eps);
}

// ---- fp32 -> (tf32 hi, tf32 lo) split for 3xTF32 library GEMMs (tf32_split.cuh) ----
__global__ void __launch_bounds__(256) u2c_split_tf32_kernel(const float4* __restrict__ x, float4* __restrict__ hi, float4* __restrict__ lo,
                                                             size_t n4, const float* __restrict__ xt, float* __restrict__ hit,
                                                             float* __restrict__ lot, int tail) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        const float4 v = x[i];
        float4 h, l;
        tf32_split(v.x, h.x, l.x); tf32_split(v.y, h.y, l.y); tf32_split(v.z, h.z, l.z); tf32_split(v.w, h.w, l.w);
        hi[i] = h; lo[i] = l;
    }
    if (blockIdx.x == 0 && (int)threadIdx.x < tail) {
        float h, l;
        tf32_split(xt[threadIdx.x], h, l);
        hit[threadIdx.x] = h; lot[threadIdx.x] = l;
    }
}

}  // namespace

extern "C" int b2d_split_tf32(const float* x, float* hi, float* lo, size_t n, void* stream) {
    if (!x || !hi || !lo) return b2d::fail(B2D_ERR_NULL, "split_tf32: null pointer");
    if (n == 0) return 0;
    if (!b2d::aligned16(x) || !b2d::aligned16(hi) || !b2d::aligned16(lo)) return b2d::fail(B2D_ERR_ALIGN, "split_tf32: buffers must be 16-byte aligned");
    const size_t n4 = n / 4;
    const int tail = (int)(n - n4 * 4);
    size_t gx = (n4 + 255) / 256;
    if (gx > b2d::num_sms() * 16) gx = b2d::num_sms() * 16;
    if (gx == 0) gx = 1;
    u2c_split_tf32_kernel<<<(unsigned)gx, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(hi),
                                                                          reinterpret_cast<float4*>(lo), n4, x + n4 * 4, hi + n4 * 4,
                                                                          lo + n4 * 4, tail);
    return b2d::check_launch("split_tf32");
}

extern "C" int b2d_u2c_embed(float* x, const float* f0, const float* phase, const float* volume, const float* embed_table,
                             const float* spk, int spk_rows, const float* aug_shift, int B, int T, void* stream) {
    if (!x || !f0 || !phase || !volume || !embed_table) return b2d::fail(B2D_ERR_NULL, "u2c_embed: null pointer");
    if (B <= 0 || T <= 0 || (spk && spk_rows != 1 && spk_rows != B)) return b2d::fail(B2D_ERR_SHAPE, "u2c_embed: bad shape");
    const int n = B * T;
    u2c_embed_kernel<<<min(n, b2d::num_sms() * 8), 256, 0, (cudaStream_t)stream>>>(x, f0, phase, volume, embed_table, spk, spk_rows, aug_shift, n, T);
    return b2d::check_launch("u2c_embed");
}

extern "C" int b2d_u2c_groupnorm_lrelu(float* x, int B, int T, int C, int groups, const float* gamma, const float* beta, float eps,
                                       float slope, double* stats_ws, void* stream) {
    if (!x || !gamma || !beta || !stats_ws) return b2d::fail(B2D_ERR_NULL, "u2c_groupnorm: null pointer");
    if (B <= 0 || T <= 0 || C != 256 || groups <= 0 || C % groups || B > 65535) return b2d::fail(B2D_ERR_SHAPE, "u2c_groupnorm: needs C = 256");
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(stats_ws, 0, (size_t)B * groups * 2 * sizeof(double), st);
    if (e != cudaSuccess) return b2d::fail((int)e, "u2c_groupnorm: memset: %s", cudaGetErrorString(e));
    const int gx = min(T, 64);
    u2c_gn_stats_kernel<<<dim3(gx, B), C, 0, st>>>(x, T, C, groups, stats_ws);
    u2c_gn_apply_kernel<<<dim3(min(T, 128), B), C, 0, st>>>(x, T, C, groups, stats_ws, gamma, beta, eps, slope);
    return b2d::check_launch("u2c_groupnorm");
}

extern "C" int b2d_u2c_layernorm(const float* x, float* y, int n_tokens, int C, const float* gamma, const float* beta, float eps,
                                 void* stream) {
    if (!x || !y || !gamma || !beta) return b2d::fail(B2D_ERR_NULL, "u2c_layernorm: null pointer");
    if (n_tokens <= 0 || C <= 0 || C % 32 || C > 1024) return b2d::fail(B2D_ERR_SHAPE, "u2c_layernorm: C must be a multiple of 32, <= 1024");
    u2c_layernorm_kernel<<<(n_tokens + 7) / 8, 256, 0, (cudaStream_t)stream>>>(x, y, n_tokens, C, gamma, beta, eps);
    return b2d::check_launch("u2c_layernorm");
}

extern "C" int b2d_u2c_glu_dwconv_silu(const float* in, const float* weight, const float* bias, float* out, int B, int T,
                                       int inner_channels, int kernel_size, void* stream) {
    if (!in || !weight || !bias || !out) return b2d::fail(B2D_ERR_NULL, "u2c_glu_dwconv: null pointer");
    if (B <= 0 || T <= 0 || inner_channels % 128 || kernel_size != kDwK || B > 65535)
        return b2d::fail(B2D_ERR_SHAPE, "u2c_glu_dwconv: needs kernel size 31 and channels multiple of 128");
    dim3 grid((T + kDwTile - 1) / kDwTile, inner_channels / 128, B);
    u2c_glu_dwconv_silu_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(in, weight, bias, out, T, inner_channels);
    return b2d::check_launch("u2c_glu_dwconv");
}

extern "C" int b2d_u2c_softmax_features(float* projected, const float* data, int rows, int n_features, int dim_head, int is_query,
                                        float eps, void* stream) {
    if (!projected || !data) return b2d::fail(B2D_ERR_NULL, "u2c_softmax_features: null pointer");
    if (rows <= 0 || n_features <= 0 || dim_head <= 0) return b2d::fail(B2D_ERR_SHAPE, "u2c_softmax_features: bad shape");
    u2c_softmax_feat_kernel<<<(rows + 7) / 8, 256, 0, (cudaStream_t)stream>>>(projected, data, rows, n_features, dim_head, is_query, eps);
    return b2d::check_launch("u2c_softmax_features");
}
