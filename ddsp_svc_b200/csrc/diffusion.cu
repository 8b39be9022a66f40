// Fused stages of the diffusion models' sampler: GaussianDiffusion (diffusion/diffusion.py:216-384) with its five
// samplers around the WaveNet denoiser (diffusion/wavenet.py).  The denoiser's products (input projection, each layer's
// k = 3 dilated convolution as ONE GEMM over a [tokens, 3 C] operand, each layer's output projection, the skip and output
// projections) are library GEMMs issued by the host side (ddsp_svc_b200/diffusion.py); these kernels are everything
// between those GEMMs:
//
//   df_layer   h = ReLU(G + b) (input projection), or r = G + b, h = (h + r[:C]) / sqrt 2, skip (+)= r[C:] (a layer's
//              residual); then the next layer's convolution operand [y[t-1] | y[t] | y[t+1]] of y = h + step, zero
//              outside the utterance, or after the last layer skip / sqrt(n_layers) for the skip projection
//   df_gate    z = G + cond_row (the condition projection with both biases folded in), sigmoid(z[:C]) tanh(z[C:])
//   df_relu    ReLU(G + b): the skip projection's activation
//   df_update  eps = G + b_out; d = a_x x + a_e eps; x' = c_x x + c_d d + c_1 h1 + c_2 h2 + c_3 h3 + c_n noise, the
//              one sampler step of DPM-Solver++, UniPC, PNDM, DDIM and DDPM with coefficients the host computes per step
//
// Activations are token-major [B, T, C] fp32.  Every kernel that feeds a GEMM writes the GEMM's operand: fp32 (lo NULL)
// or the TF32 (hi, lo) halves of a 3xTF32 product.  Each output element has exactly one writing thread (the convolution
// operand is scattered from its source token, never gathered from neighbours that the same launch updates): no atomics,
// no shared memory, results are bit-identical from run to run.
#ifndef B2D_HOST_EMU               // tests/emu/ runs these kernels' source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif
#include "tf32_split.cuh"

namespace {

__device__ __forceinline__ void df_emit4(const float (&v)[4], float* __restrict__ hi, float* __restrict__ lo, size_t i) {
    for (int k = 0; k < 4; ++k) tf32_emit(v[k], hi, lo, i + k);
}

// G: [n_tokens, C] (stage 0) or [n_tokens, 2 C] (stages 1, 2: a layer's output projection); h, skip [n_tokens, C].
// stage 0: h = ReLU(G + b) (wavenet.py:91-94).  stage 1 (layer 0) / 2 (later layers): r = G + b, h = (h + r[:C]) / sqrt 2,
// skip = r[C:] / skip += r[C:] (wavenet.py:60-62, :100-102).  Then with step: the convolution operand [n_tokens, 3 C]
// of y = h + step[b] (wavenet.py:48): token n's y goes to row n block 1, row n + 1 block 0 and row n - 1 block 2 when
// those rows are in the same utterance; the blocks that would read across an utterance's edge are written as zeros by
// the edge token itself.  Without step (after the last layer): skip / skip_div into the [n_tokens, C] operand.
// One thread per 4 channels of one token.
__global__ void __launch_bounds__(256) df_layer_kernel(const float4* __restrict__ g, const float4* __restrict__ bias,
                                                       float4* __restrict__ h, float4* __restrict__ skip, int stage,
                                                       const float* __restrict__ step, int step_stride, float skip_div,
                                                       int T, int C4, size_t n4, float* __restrict__ hi,
                                                       float* __restrict__ lo) {
    const float kSqrt2 = 1.41421356237309515f;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        const size_t tok = i / C4;
        const int c4 = (int)(i - tok * C4);
        float r[4], s[4] = {0.f, 0.f, 0.f, 0.f};
        if (stage == 0) {
            const float4 gv = g[i], bv = __ldg(bias + c4);
            r[0] = fmaxf(gv.x + bv.x, 0.f); r[1] = fmaxf(gv.y + bv.y, 0.f);
            r[2] = fmaxf(gv.z + bv.z, 0.f); r[3] = fmaxf(gv.w + bv.w, 0.f);
        } else {
            const size_t row = tok * 2 * C4;
            const float4 gr = g[row + c4], br = __ldg(bias + c4), gs = g[row + C4 + c4], bs = __ldg(bias + C4 + c4);
            const float4 hv = h[i];
            r[0] = (hv.x + (gr.x + br.x)) / kSqrt2; r[1] = (hv.y + (gr.y + br.y)) / kSqrt2;
            r[2] = (hv.z + (gr.z + br.z)) / kSqrt2; r[3] = (hv.w + (gr.w + br.w)) / kSqrt2;
            s[0] = gs.x + bs.x; s[1] = gs.y + bs.y; s[2] = gs.z + bs.z; s[3] = gs.w + bs.w;
            if (stage == 2) {
                const float4 sv = skip[i];
                s[0] = sv.x + s[0]; s[1] = sv.y + s[1]; s[2] = sv.z + s[2]; s[3] = sv.w + s[3];
            }
            skip[i] = make_float4(s[0], s[1], s[2], s[3]);
        }
        h[i] = make_float4(r[0], r[1], r[2], r[3]);
        if (step) {
            const size_t b = tok / T;
            const int t = (int)(tok - b * T);
            const float4 sv = *reinterpret_cast<const float4*>(step + b * step_stride + 4 * c4);
            const float y[4] = {r[0] + sv.x, r[1] + sv.y, r[2] + sv.z, r[3] + sv.w};
            const float zero[4] = {0.f, 0.f, 0.f, 0.f};
            const size_t C = 4 * (size_t)C4, row3 = tok * 3 * C + 4 * (size_t)c4;
            df_emit4(y, hi, lo, row3 + C);                                      // row n, tap at t
            if (t + 1 < T) df_emit4(y, hi, lo, row3 + 3 * C);                    // row n + 1, tap at t - 1
            else df_emit4(zero, hi, lo, row3 + 2 * C);                           // row n, tap at t + 1: padding
            if (t > 0) df_emit4(y, hi, lo, row3 - 3 * C + 2 * C);                // row n - 1, tap at t + 1
            else df_emit4(zero, hi, lo, row3);                                   // row n, tap at t - 1: padding
        } else {
            const float o[4] = {s[0] / skip_div, s[1] / skip_div, s[2] / skip_div, s[3] / skip_div};
            df_emit4(o, hi, lo, 4 * i);
        }
    }
}

// G [n_tokens, 2 C] (the convolution), cond row n at cond + n cond_stride (2 C columns): z = G + cond,
// sigmoid(z[:C]) tanh(z[C:]) into the [n_tokens, C] operand (wavenet.py:50-56).  One thread per 4 channels.
__global__ void __launch_bounds__(256) df_gate_kernel(const float4* __restrict__ g, const float* __restrict__ cond,
                                                      int cond_stride, int C4, size_t n4, float* __restrict__ hi,
                                                      float* __restrict__ lo) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        const size_t tok = i / C4;
        const int c4 = (int)(i - tok * C4);
        const float4 ga = g[tok * 2 * C4 + c4], gb = g[tok * 2 * C4 + C4 + c4];
        const float* crow = cond + tok * cond_stride;
        const float4 ca = *reinterpret_cast<const float4*>(crow + 4 * c4);
        const float4 cb = *reinterpret_cast<const float4*>(crow + 4 * (C4 + c4));
        const float za[4] = {ga.x + ca.x, ga.y + ca.y, ga.z + ca.z, ga.w + ca.w};
        const float zb[4] = {gb.x + cb.x, gb.y + cb.y, gb.z + cb.z, gb.w + cb.w};
        float o[4];
        for (int k = 0; k < 4; ++k) o[k] = (1.0f / (1.0f + expf(-za[k]))) * tanhf(zb[k]);
        df_emit4(o, hi, lo, 4 * i);
    }
}

// ReLU(G + b) over [n_tokens, C] into the operand (wavenet.py:103-104).  One thread per 4 channels.
__global__ void __launch_bounds__(256) df_relu_kernel(const float4* __restrict__ g, const float4* __restrict__ bias,
                                                      int C4, size_t n4, float* __restrict__ hi, float* __restrict__ lo) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        const float4 gv = g[i], bv = __ldg(bias + (int)(i % C4));
        const float o[4] = {fmaxf(gv.x + bv.x, 0.f), fmaxf(gv.y + bv.y, 0.f), fmaxf(gv.z + bv.z, 0.f),
                            fmaxf(gv.w + bv.w, 0.f)};
        df_emit4(o, hi, lo, 4 * i);
    }
}

// One sampler step over [n_tokens, M] (see the file comment); coef [8] = a_x, a_e, c_x, c_d, c_1, c_2, c_3, c_n on the
// device.  h1..h3 token-major [n_tokens, M] or NULL; noise channel-major [B, 1, M, T] or NULL; d_out (may be one of
// h1..h3: each element is read before it is overwritten by the same thread) and x_out (may be x) optional; hi NULL: no
// operand.  Not __restrict__: the in-place aliases are part of the contract.
__global__ void __launch_bounds__(256) df_update_kernel(const float* __restrict__ g, const float* __restrict__ bias,
                                                        const float* __restrict__ coef, const float* x, float* d_out,
                                                        const float* h1, const float* h2, const float* h3,
                                                        const float* __restrict__ noise, int T, int M, size_t n,
                                                        float* x_out, float* __restrict__ hi, float* __restrict__ lo) {
    const float a_x = __ldg(coef + 0), a_e = __ldg(coef + 1), c_x = __ldg(coef + 2), c_d = __ldg(coef + 3);
    const float c_1 = __ldg(coef + 4), c_2 = __ldg(coef + 5), c_3 = __ldg(coef + 6), c_n = __ldg(coef + 7);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t tok = i / M;
        const int m = (int)(i - tok * M);
        const float eps = g[i] + __ldg(bias + m);
        const float xv = x[i];
        const float d = a_x * xv + a_e * eps;
        float v = c_x * xv + c_d * d;
        if (h1) v += c_1 * h1[i];
        if (h2) v += c_2 * h2[i];
        if (h3) v += c_3 * h3[i];
        if (noise) {
            const size_t b = tok / T;
            const int t = (int)(tok - b * T);
            v += c_n * noise[(b * M + m) * T + t];
        }
        if (d_out) d_out[i] = d;
        if (x_out) x_out[i] = v;
        if (hi) tf32_emit(v, hi, lo, i);
    }
}

}  // namespace

#ifndef B2D_HOST_EMU
namespace {
unsigned df_grid(size_t work) {
    size_t g = (work + 255) / 256;
    const size_t cap = (size_t)b2d::num_sms() * 8;
    return (unsigned)(g < 1 ? 1 : g > cap ? cap : g);
}
}  // namespace

extern "C" int b2d_df_layer(const float* g, const float* bias, float* h, float* skip, int stage, const float* step,
                            int step_stride, float skip_div, int B, int T, int C, float* hi, float* lo, void* stream) {
    if (!g || !bias || !h || !hi || (stage > 0 && !skip)) return b2d::fail(B2D_ERR_NULL, "df_layer: null pointer");
    if (B <= 0 || T <= 0 || C <= 0 || (step && step_stride != 0 && step_stride < C) || (!step && !(skip_div > 0.f)))
        return b2d::fail(B2D_ERR_SHAPE, "df_layer: bad shape");
    if (stage < 0 || stage > 2 || (stage == 0 && !step))
        return b2d::fail(B2D_ERR_UNSUPPORTED, "df_layer: stage must be 0 (input, with step), 1 or 2 (residual)");
    if (C % 4 || !b2d::aligned16(g) || !b2d::aligned16(bias) || !b2d::aligned16(h) || (skip && !b2d::aligned16(skip)) ||
        (step && (step_stride % 4 || !b2d::aligned16(step))))
        return b2d::fail(B2D_ERR_ALIGN, "df_layer: width, stride and buffers must be 16-byte multiples");
    const size_t n4 = (size_t)B * T * (C / 4);
    df_layer_kernel<<<df_grid(n4), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float4*>(g), reinterpret_cast<const float4*>(bias), reinterpret_cast<float4*>(h),
        reinterpret_cast<float4*>(skip), stage, step, step_stride, skip_div, T, C / 4, n4, hi, lo);
    return b2d::check_launch("df_layer");
}

extern "C" int b2d_df_gate(const float* g, const float* cond, int cond_stride, int n_tokens, int C, float* hi, float* lo,
                           void* stream) {
    if (!g || !cond || !hi) return b2d::fail(B2D_ERR_NULL, "df_gate: null pointer");
    if (n_tokens <= 0 || C <= 0 || cond_stride < 2 * C) return b2d::fail(B2D_ERR_SHAPE, "df_gate: bad shape");
    if (C % 4 || cond_stride % 4 || !b2d::aligned16(g) || !b2d::aligned16(cond))
        return b2d::fail(B2D_ERR_ALIGN, "df_gate: width, stride and buffers must be 16-byte multiples");
    const size_t n4 = (size_t)n_tokens * (C / 4);
    df_gate_kernel<<<df_grid(n4), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(g), cond, cond_stride,
                                                                  C / 4, n4, hi, lo);
    return b2d::check_launch("df_gate");
}

extern "C" int b2d_df_relu(const float* g, const float* bias, int n_tokens, int C, float* hi, float* lo, void* stream) {
    if (!g || !bias || !hi) return b2d::fail(B2D_ERR_NULL, "df_relu: null pointer");
    if (n_tokens <= 0 || C <= 0) return b2d::fail(B2D_ERR_SHAPE, "df_relu: bad shape");
    if (C % 4 || !b2d::aligned16(g) || !b2d::aligned16(bias))
        return b2d::fail(B2D_ERR_ALIGN, "df_relu: width and buffers must be 16-byte multiples");
    const size_t n4 = (size_t)n_tokens * (C / 4);
    df_relu_kernel<<<df_grid(n4), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(g),
                                                                  reinterpret_cast<const float4*>(bias), C / 4, n4, hi, lo);
    return b2d::check_launch("df_relu");
}

extern "C" int b2d_df_update(const float* g, const float* bias, const float* coef, const float* x, float* d_out,
                             const float* h1, const float* h2, const float* h3, const float* noise, int B, int T, int M,
                             float* x_out, float* hi, float* lo, void* stream) {
    if (!g || !bias || !coef || !x || (lo && !hi)) return b2d::fail(B2D_ERR_NULL, "df_update: null pointer");
    if (B <= 0 || T <= 0 || M <= 0) return b2d::fail(B2D_ERR_SHAPE, "df_update: bad shape");
    const size_t n = (size_t)B * T * M;
    df_update_kernel<<<df_grid(n), 256, 0, (cudaStream_t)stream>>>(g, bias, coef, x, d_out, h1, h2, h3, noise, T, M, n,
                                                                   x_out, hi, lo);
    return b2d::check_launch("df_update");
}
#endif  // B2D_HOST_EMU
