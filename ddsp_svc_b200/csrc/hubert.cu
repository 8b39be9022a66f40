// The HuBERT / ContentVec units encoder (encoder/hubert/model.py, fairseq's HubertModel), inference.  The linear layers
// (the feature convolutions 1-6 as row-pair GEMMs, the feature projection, QKV, out-proj, the FFN and `proj`) run on the
// library GEMMs in 3xTF32; these kernels do everything between them:
//
//   hb_conv0     Conv1d(1 -> 512, k 10, s 5, no bias) in direct fp32, the zero pad of HubertSoft.units applied by index.
//                A CTA owns 64 frames x 512 channels of one utterance; besides the output it writes its fp64 partial
//                sums of x and x^2 per channel for the GroupNorm(512, 512) statistics.  Rows past the valid length are
//                written as zeros.
//   hb_gn_finalize  the partials of one (utterance, channel) summed in tile order -> GroupNorm scale and shift.
//   hb_act       elementwise: optional per-(utterance, channel) affine, exact-erf GELU, written as the next GEMM's
//                operand (fp32, or its TF32 halves).
//   hb_ln        one warp per token: LayerNorm(C) of x (+ y), optionally GELU first (the last feature convolution
//                followed by feature_projection.norm), written in fp32 and / or as the next GEMM's operand.  Input
//                rows are gathered from a [B, rows_per_b, C] buffer, so the padded feature rows are dropped here.
//   hb_posconv   the grouped positional convolution Conv1d(768, 768, 128, padding 64, groups 16) with the last output
//                frame dropped, + bias, GELU.  A CTA owns (utterance, group, 64 frames): the 191-row halo of the
//                group's 48 channels is staged once, the folded weights stream through shared memory 8 taps at a time.
//                fp32 FMA.
//   hb_attention non-causal softmax attention, 12 heads x 64, flash style: a CTA owns (utterance, head, 64 queries),
//                streams 64-key tiles of K and V through shared memory and keeps the online-softmax state (max, sum)
//                and the output accumulator in registers; keys past T are masked.  fp32 FMA, expf.  The output is
//                written as the out-projection's operand.
//   hb_align     the frame gather of Units_Encoder.encode: row min(rint(ratio * i), T - 1), the index a float32
//                product rounded half to even, as torch computes it.
//
// No atomics: every output element has one writer and a fixed summation order, so results are bit-identical from run
// to run.
#ifndef B2D_HOST_EMU               // tests/emu/ runs these kernels' source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif
#include "tf32_split.cuh"

namespace {

constexpr int kC0 = 512;                     // feature-extractor channels
constexpr int kD = 768;                      // model width
constexpr int kConv0Tile = 64;               // hb_conv0 frames per CTA
constexpr int kPosGroups = 16, kPosCh = 48, kPosTaps = 128, kPosPad = 64;
constexpr int kPosBM = 64, kPosKC = 8, kPosHalo = kPosBM + kPosTaps - 1, kPosLd = kPosCh + 1;
constexpr int kPosXs = (kPosHalo * kPosLd + 3) / 4 * 4;          // the weight chunk after it stays 16-byte aligned
constexpr size_t kPosSmem = (size_t)(kPosXs + kPosKC * kPosCh * kPosCh) * sizeof(float);
constexpr int kHeads = 12, kHd = 64, kAttnQ = 64, kAttnK = 64;
constexpr size_t kAttnSmem = (size_t)(kAttnQ * kHd + kAttnK * (kHd + 1) + kAttnK * kHd + 4 * 16 * kAttnK) * sizeof(float);

__device__ __forceinline__ float hb_gelu(float x) { return (x * 0.5f) * (1.0f + erff(x * 0.70710678118654752f)); }

// ---- hb_conv0 ----------------------------------------------------------------------------------------------------------
// x [B, N] -> y [B, La, 512] (rows >= L0 zero), part [B, n_tiles, 2, 512] fp64 (sum, sum of squares over valid rows)
__global__ void __launch_bounds__(256) hb_conv0_kernel(const float* __restrict__ x, int N, int pad,
                                                       const float* __restrict__ w, int L0, int La,
                                                       float* __restrict__ y, double* __restrict__ part) {
    B2D_SHARED(float, s, [5 * (kConv0Tile - 1) + 10]);
    const int tile = blockIdx.x, b = blockIdx.y, t0 = tile * kConv0Tile;
    const int n_tiles = gridDim.x;
    const float* xb = x + (size_t)b * N;
    for (int i = threadIdx.x; i < 5 * (kConv0Tile - 1) + 10; i += blockDim.x) {
        const int n = 5 * t0 + i - pad;
        s[i] = (n >= 0 && n < N) ? xb[n] : 0.f;
    }
    float wr[2][10];
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int k = 0; k < 10; ++k) wr[j][k] = w[(threadIdx.x + 256 * j) * 10 + k];
    __syncthreads();
    double sum[2] = {0.0, 0.0}, sq[2] = {0.0, 0.0};
    for (int tt = 0; tt < kConv0Tile; ++tt) {
        const int t = t0 + tt;
        if (t >= La) break;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            float acc = 0.f;
            if (t < L0) {
#pragma unroll
                for (int k = 0; k < 10; ++k) acc = fmaf(wr[j][k], s[5 * tt + k], acc);
                sum[j] += (double)acc;
                sq[j] += (double)acc * (double)acc;
            }
            y[((size_t)b * La + t) * kC0 + threadIdx.x + 256 * j] = acc;
        }
    }
    double* p = part + ((size_t)b * n_tiles + tile) * 2 * kC0;
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        p[threadIdx.x + 256 * j] = sum[j];
        p[kC0 + threadIdx.x + 256 * j] = sq[j];
    }
}

// part [B, n_tiles, 2, 512] -> scale, shift [B, 512]: GroupNorm(512, 512) over the L0 valid frames, biased variance
__global__ void __launch_bounds__(256) hb_gn_finalize_kernel(const double* __restrict__ part, int B, int n_tiles, int L0,
                                                             const float* __restrict__ gamma,
                                                             const float* __restrict__ beta, float eps,
                                                             float* __restrict__ scale, float* __restrict__ shift) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * kC0) return;
    const int b = i / kC0, c = i % kC0;
    double s = 0.0, q = 0.0;
    for (int t = 0; t < n_tiles; ++t) {
        const double* p = part + ((size_t)b * n_tiles + t) * 2 * kC0;
        s += p[c];
        q += p[kC0 + c];
    }
    const double mean = s / L0, var = fmax(q / L0 - mean * mean, 0.0);
    const double sc = (double)gamma[c] / sqrt(var + (double)eps);
    scale[i] = (float)sc;
    shift[i] = (float)((double)beta[c] - mean * sc);
}

// ---- hb_act ------------------------------------------------------------------------------------------------------------
// x [B rows_per_b, C] -> GELU(x scale[b, c] + shift[b, c]) (affine when scale != NULL) as an operand
__global__ void __launch_bounds__(256) hb_act_kernel(const float* __restrict__ x, size_t n, int C, int rows_per_b,
                                                     const float* __restrict__ scale, const float* __restrict__ shift,
                                                     float* __restrict__ hi, float* __restrict__ lo) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        float v = x[i];
        if (scale) {
            const size_t row = i / C;
            const size_t bc = (row / rows_per_b) * C + i % C;
            v = fmaf(v, scale[bc], shift[bc]);
        }
        tf32_emit(hb_gelu(v), hi, lo, i);
    }
}

// ---- hb_ln -------------------------------------------------------------------------------------------------------------
// row r < B T: v = x[(r / T) rows_per_b + r % T] (+ y[r]); optionally GELU(v); LayerNorm over C = 32 NPL channels
// -> h[r] (when h != NULL) and the operand (hi, lo) at r (when hi != NULL).  h may alias x when rows_per_b == T.
template <int NPL>
__global__ void __launch_bounds__(256) hb_ln_kernel(const float* x, const float* __restrict__ y, int rows, int T,
                                                    int rows_per_b, int gelu, const float* __restrict__ gamma,
                                                    const float* __restrict__ beta, float eps, float* h,
                                                    float* __restrict__ hi, float* __restrict__ lo) {
    constexpr int C = 32 * NPL;
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    if (r >= rows) return;
    const float* xr = x + ((size_t)(r / T) * rows_per_b + r % T) * C;
    float v[NPL];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
        const int c = lane + 32 * j;
        float a = xr[c];
        if (y) a += y[(size_t)r * C + c];
        if (gelu) a = hb_gelu(a);
        v[j] = a;
        s += a;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / C;
    float q = 0.f;
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
        const float d = v[j] - mean;
        q = fmaf(d, d, q);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q / C + eps);
    __syncwarp();                                     // every lane has read its row before h (possibly x) is written
#pragma unroll
    for (int j = 0; j < NPL; ++j) {
        const int c = lane + 32 * j;
        const float o = fmaf((v[j] - mean) * rstd, gamma[c], beta[c]);
        const size_t i = (size_t)r * C + c;
        if (h) h[i] = o;
        tf32_emit_opt(o, hi, lo, i);
    }
}

// ---- hb_posconv --------------------------------------------------------------------------------------------------------
// x [B T, 768], w [16][128][48 ci][48 co] (weight norm folded), bias [768] -> y [B T, 768] = GELU(conv + bias)
__global__ void __launch_bounds__(256) hb_posconv_kernel(const float* __restrict__ x, int T,
                                                         const float* __restrict__ w, const float* __restrict__ bias,
                                                         float* __restrict__ y) {
    extern __shared__ float4 smem4[];
    float* xs = reinterpret_cast<float*>(smem4);               // [kPosHalo][kPosLd]
    float* ws = xs + kPosXs;                                   // [kPosKC][48 ci][48 co]
    const int t0 = blockIdx.x * kPosBM, g = blockIdx.y, b = blockIdx.z;
    const int tid = threadIdx.x, tg = tid / 16, cg = tid % 16;
    for (int i = tid; i < kPosHalo * kPosCh; i += blockDim.x) {
        const int row = i / kPosCh, ci = i % kPosCh, t = t0 + row - kPosPad;
        xs[row * kPosLd + ci] = (t >= 0 && t < T) ? x[((size_t)b * T + t) * kD + g * kPosCh + ci] : 0.f;
    }
    float acc[4][3];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) acc[i][j] = 0.f;
    const float4* wg = reinterpret_cast<const float4*>(w + (size_t)g * kPosTaps * kPosCh * kPosCh);
    constexpr int kChunk4 = kPosKC * kPosCh * kPosCh / 4;
    for (int k0 = 0; k0 < kPosTaps; k0 += kPosKC) {
        __syncthreads();                                       // the previous chunk is consumed (and xs is staged)
        for (int i = tid; i < kChunk4; i += blockDim.x) reinterpret_cast<float4*>(ws)[i] = wg[(size_t)k0 / kPosKC * kChunk4 + i];
        __syncthreads();
        for (int kk = 0; kk < kPosKC; ++kk) {
            const float* xk = xs + (tg * 4 + k0 + kk) * kPosLd;
            const float* wk = ws + kk * kPosCh * kPosCh + cg * 3;
#pragma unroll 4
            for (int ci = 0; ci < kPosCh; ++ci) {
                float xv[4], wv[3];
#pragma unroll
                for (int i = 0; i < 4; ++i) xv[i] = xk[i * kPosLd + ci];
#pragma unroll
                for (int j = 0; j < 3; ++j) wv[j] = wk[ci * kPosCh + j];
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 3; ++j) acc[i][j] = fmaf(xv[i], wv[j], acc[i][j]);
            }
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int t = t0 + tg * 4 + i;
        if (t >= T) continue;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const int co = g * kPosCh + cg * 3 + j;
            y[((size_t)b * T + t) * kD + co] = hb_gelu(acc[i][j] + bias[co]);
        }
    }
}

// ---- hb_attention ------------------------------------------------------------------------------------------------------
// qkv [B T, 3 768] (q | k | v, head h at columns h 64) -> o [B T, 768] = softmax(q k^T / 8) v per head, as an operand
__global__ void __launch_bounds__(128, 1) hb_attention_kernel(const float* __restrict__ qkv, int T,
                                                           float* __restrict__ hi, float* __restrict__ lo) {
    extern __shared__ float4 smem4[];
    auto qs = reinterpret_cast<float (*)[kHd]>(smem4);                         // [kAttnQ][kHd]
    auto ks = reinterpret_cast<float (*)[kHd + 1]>(&qs[kAttnQ][0]);            // [kAttnK][kHd + 1]
    auto vs = reinterpret_cast<float (*)[kHd]>(&ks[kAttnK][0]);                // [kAttnK][kHd]
    auto ps = reinterpret_cast<float (*)[16][kAttnK]>(&vs[kAttnK][0]);         // [4 warps][16][kAttnK]
    const int q0 = blockIdx.x * kAttnQ, head = blockIdx.y, b = blockIdx.z;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const size_t ld = 3 * kD;
    const float* base = qkv + (size_t)b * T * ld + head * kHd;
    for (int i = tid; i < kAttnQ * kHd; i += blockDim.x) {
        const int r = i / kHd, d = i % kHd, t = q0 + r;
        qs[r][d] = t < T ? base[(size_t)t * ld + d] * 0.125f : 0.f;      // 1 / sqrt(64): exact
    }
    float o[16][2], m[16], l[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        o[i][0] = o[i][1] = 0.f;
        m[i] = -INFINITY;
        l[i] = 0.f;
    }
    for (int k0 = 0; k0 < T; k0 += kAttnK) {
        __syncthreads();                                       // the previous tile is consumed
        for (int i = tid; i < kAttnK * kHd; i += blockDim.x) {
            const int r = i / kHd, d = i % kHd, t = k0 + r;
            const bool in = t < T;
            ks[r][d] = in ? base[(size_t)t * ld + kD + d] : 0.f;
            vs[r][d] = in ? base[(size_t)t * ld + 2 * kD + d] : 0.f;
        }
        __syncthreads();
        float s[16][2];
#pragma unroll
        for (int i = 0; i < 16; ++i) s[i][0] = s[i][1] = 0.f;
        for (int d = 0; d < kHd; ++d) {
            const float ka = ks[lane][d], kb = ks[lane + 32][d];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const float q = qs[warp * 16 + i][d];
                s[i][0] = fmaf(q, ka, s[i][0]);
                s[i][1] = fmaf(q, kb, s[i][1]);
            }
        }
        const bool va = k0 + lane < T, vb = k0 + lane + 32 < T;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const float sa = va ? s[i][0] : -INFINITY, sb = vb ? s[i][1] : -INFINITY;
            float mx = fmaxf(sa, sb);
#pragma unroll
            for (int off = 16; off; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
            const float mn = fmaxf(m[i], mx);                  // finite: key k0 is always valid
            const float alpha = expf(m[i] - mn);
            const float pa = expf(sa - mn), pb = expf(sb - mn);
            float ps_sum = pa + pb;
#pragma unroll
            for (int off = 16; off; off >>= 1) ps_sum += __shfl_xor_sync(0xffffffffu, ps_sum, off);
            l[i] = fmaf(l[i], alpha, ps_sum);
            m[i] = mn;
            o[i][0] *= alpha;
            o[i][1] *= alpha;
            ps[warp][i][lane] = pa;
            ps[warp][i][lane + 32] = pb;
        }
        __syncwarp();
        for (int k = 0; k < kAttnK; ++k) {
            const float va_ = vs[k][lane], vb_ = vs[k][lane + 32];
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const float p = ps[warp][i][k];
                o[i][0] = fmaf(p, va_, o[i][0]);
                o[i][1] = fmaf(p, vb_, o[i][1]);
            }
        }
        __syncwarp();
    }
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int t = q0 + warp * 16 + i;
        if (t >= T) continue;
        const float inv = 1.f / l[i];
        const size_t row = ((size_t)b * T + t) * kD + head * kHd;
        tf32_emit(o[i][0] * inv, hi, lo, row + lane);
        tf32_emit(o[i][1] * inv, hi, lo, row + lane + 32);
    }
}

// ---- hb_align ----------------------------------------------------------------------------------------------------------
// units [B, T, C] -> out [B, n_frames, C]: row min(rint(ratio i), T - 1) (ratio i a float32 product)
__global__ void __launch_bounds__(256) hb_align_kernel(const float* __restrict__ units, int B, int T, int C,
                                                       float ratio, int n_frames, float* __restrict__ out) {
    const size_t n = (size_t)B * n_frames * C;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const size_t bf = i / C;
        const int f = (int)(bf % n_frames), b = (int)(bf / n_frames);
        const float idx = rintf(__fmul_rn(ratio, (float)f));
        const int t = idx >= (float)(T - 1) ? T - 1 : (int)idx;
        out[i] = units[((size_t)b * T + t) * C + c];
    }
}

#ifndef B2D_HOST_EMU
unsigned hb_grid(size_t n) {
    const size_t blocks = (n + 255) / 256, cap = (size_t)b2d::num_sms() * 16;
    return (unsigned)(blocks < cap ? (blocks ? blocks : 1) : cap);
}
#endif  // B2D_HOST_EMU

}  // namespace

#ifndef B2D_HOST_EMU
namespace b2d {

int hubert_conv0_launch(const float* x, int B, int N, int pad, const float* w, int L0, int La, float* y, double* part,
                        cudaStream_t stream) {
    const dim3 grid((La + kConv0Tile - 1) / kConv0Tile, B);
    hb_conv0_kernel<<<grid, 256, 0, stream>>>(x, N, pad, w, L0, La, y, part);
    return check_launch("hubert_conv0");
}

int hubert_gn_finalize_launch(const double* part, int B, int n_tiles, int L0, const float* gamma, const float* beta,
                              float eps, float* scale, float* shift, cudaStream_t stream) {
    hb_gn_finalize_kernel<<<(B * kC0 + 255) / 256, 256, 0, stream>>>(part, B, n_tiles, L0, gamma, beta, eps, scale,
                                                                     shift);
    return check_launch("hubert_gn_finalize");
}

int hubert_act_launch(const float* x, int rows, int C, int rows_per_b, const float* scale, const float* shift, float* hi,
                      float* lo, cudaStream_t stream) {
    const size_t n = (size_t)rows * C;
    hb_act_kernel<<<hb_grid(n), 256, 0, stream>>>(x, n, C, rows_per_b, scale, shift, hi, lo);
    return check_launch("hubert_act");
}

int hubert_ln_launch(const float* x, const float* y, int rows, int T, int rows_per_b, int C, int gelu,
                     const float* gamma, const float* beta, float eps, float* h, float* hi, float* lo,
                     cudaStream_t stream) {
    const unsigned grid = (unsigned)((rows + 7) / 8);
    if (C == 512)
        hb_ln_kernel<16><<<grid, 256, 0, stream>>>(x, y, rows, T, rows_per_b, gelu, gamma, beta, eps, h, hi, lo);
    else
        hb_ln_kernel<24><<<grid, 256, 0, stream>>>(x, y, rows, T, rows_per_b, gelu, gamma, beta, eps, h, hi, lo);
    return check_launch("hubert_ln");
}

int hubert_posconv_launch(const float* x, int B, int T, const float* w, const float* bias, float* y,
                          cudaStream_t stream) {
    // the opt-in is set on every call (one configuration), so concurrent host threads never see it lower
    cudaError_t e = cudaFuncSetAttribute(hb_posconv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPosSmem);
    if (e != cudaSuccess) return fail((int)e, "hubert_posconv: smem attr (%zu B): %s", kPosSmem, cudaGetErrorString(e));
    const dim3 grid((T + kPosBM - 1) / kPosBM, kPosGroups, B);
    hb_posconv_kernel<<<grid, 256, kPosSmem, stream>>>(x, T, w, bias, y);
    return check_launch("hubert_posconv");
}

int hubert_attention_launch(const float* qkv, int B, int T, float* hi, float* lo, cudaStream_t stream) {
    cudaError_t e = cudaFuncSetAttribute(hb_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         (int)kAttnSmem);
    if (e != cudaSuccess)
        return fail((int)e, "hubert_attention: smem attr (%zu B): %s", kAttnSmem, cudaGetErrorString(e));
    const dim3 grid((T + kAttnQ - 1) / kAttnQ, kHeads, B);
    hb_attention_kernel<<<grid, 128, kAttnSmem, stream>>>(qkv, T, hi, lo);
    return check_launch("hubert_attention");
}

int hubert_align_launch(const float* units, int B, int T, int C, float ratio, int n_frames, float* out,
                        cudaStream_t stream) {
    hb_align_kernel<<<hb_grid((size_t)B * n_frames * C), 256, 0, stream>>>(units, B, T, C, ratio, n_frames, out);
    return check_launch("hubert_align");
}

}  // namespace b2d
#endif  // B2D_HOST_EMU
