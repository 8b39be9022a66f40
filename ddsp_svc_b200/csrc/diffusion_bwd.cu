// The diffusion models' training loss (diffusion/diffusion.py:194-238: q_sample, the denoiser, F.mse_loss with loss_type
// 'l2') and the backward of the WaveNet denoiser (diffusion/wavenet.py).  The GEMMs and their adjoints (dX = gY W,
// dW = gY^T X), the bias column sums, the loss itself (reflow_bwd.cu's rf_loss / rf_loss_backward with w = 1 and
// target = noise) and the step sums (rf_step_sums) are issued by the host side (ddsp_svc_b200/diffusion.py); these
// kernels are everything else between them:
//
//   df_loss_input      x_t = sqrt_ac[t_b] norm(gt) + sqrt_1m_ac[t_b] noise, the coefficients gathered on the device
//   df_relu_backward   g (x > 0) with x = pre + bias (input projection, skip projection)
//   df_mish_backward   g d/dx (x tanh(softplus x)) (the step MLP)
//   df_gate_backward   g_z of sigmoid(z[:C]) tanh(z[C:]) recomputed from z = G + cond, into column block `layer` of G_Z
//   df_layer_backward  g_y = the adjoint of df_layer's k = 3 scatter, g_h = g_h' / sqrt 2 + g_y in place, the next
//                      layer's g_R = [g_h / sqrt 2 | g_skip / skip_div], per-slab sums of g_y per utterance
//
// Activations are token-major [B, T, C] fp32.  Every output that feeds a GEMM is written as its operand: fp32, plus the
// TF32 (hi, lo) halves of a 3xTF32 product when the caller asks for them.  No atomics and no shared memory.  Each output
// element has one writing thread; sums over tokens run per fixed slab of kTokenSlab frames (token_slab.cuh) of one
// utterance in fp64 (the layout rf_step_sums reads), so results do not depend on the grid and are bit-identical.
#ifndef B2D_HOST_EMU               // tests/emu/ runs these kernels' source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif
#include "tf32_split.cuh"
#include "token_slab.cuh"

namespace {

constexpr int kDfSlab = kTokenSlab;      // rf_step_sums reads these slabs: the same constant as reflow_bwd.cu's

__device__ __forceinline__ void dfb_emit(float v, float* __restrict__ hi, float* __restrict__ lo, size_t i) {
    if (!hi) return;
    if (lo) {
        float h, l;
        tf32_split(v, h, l);
        hi[i] = h;
        lo[i] = l;
    } else {
        hi[i] = v;
    }
}

// x_t over [B T, M] (gt and noise token-major, t [B] int64 on the device): the reference's fp32 association, norm as
// rf_start computes it, then two products and a sum, no contraction.  A step outside [0, n_steps) gives NaN.
__global__ void __launch_bounds__(256) df_loss_input_kernel(const float* __restrict__ gt, const float* __restrict__ noise,
                                                            const long long* __restrict__ t,
                                                            const float* __restrict__ sqrt_ac,
                                                            const float* __restrict__ sqrt_1m_ac, int n_steps,
                                                            float spec_min, float spec_range, int T, int M, size_t n,
                                                            float* __restrict__ hi, float* __restrict__ lo) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const long long s = __ldg(t + i / ((size_t)T * M));
        float v = __int_as_float(0x7fc00000);
        if (s >= 0 && s < n_steps) {
            const float x0 = ((gt[i] - spec_min) / spec_range) * 2.0f - 1.0f;          // diffusion.py:62 (norm_spec)
            v = __fadd_rn(__fmul_rn(__ldg(sqrt_ac + s), x0), __fmul_rn(__ldg(sqrt_1m_ac + s), noise[i]));
        }
        dfb_emit(v, hi, lo, i);
    }
}

// gx [n_rows, C] = gy where pre + bias[c] > 0 (the forward's ReLU(G + b) as df_layer / df_relu compute it), else 0
__global__ void __launch_bounds__(256) df_relu_bwd_kernel(const float* __restrict__ gy, const float* __restrict__ pre,
                                                          const float* __restrict__ bias, int C, size_t n,
                                                          float* __restrict__ gx, float* __restrict__ hi,
                                                          float* __restrict__ lo) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float x = pre[i] + __ldg(bias + (int)(i % C));
        const float r = x > 0.f ? gy[i] : 0.f;
        gx[i] = r;
        dfb_emit(r, hi, lo, i);
    }
}

// gx [n] = gy (tanh(sp) + x sigmoid(x) (1 - tanh(sp)^2)), sp = softplus(x) (torch's threshold 20: sp = x above it)
__global__ void __launch_bounds__(256) df_mish_bwd_kernel(const float* __restrict__ gy, const float* __restrict__ x, size_t n,
                                                          float* __restrict__ gx, float* __restrict__ hi,
                                                          float* __restrict__ lo) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float v = x[i];
        const float th = tanhf(v > 20.f ? v : log1pf(expf(v)));
        const float sg = 1.0f / (1.0f + expf(-v));
        const float r = gy[i] * (th + v * sg * (1.0f - th * th));
        gx[i] = r;
        dfb_emit(r, hi, lo, i);
    }
}

// ga [N, C] the cotangent of the gate's output; z = G + cond over [N, 2 C] as df_gate computes it (cond row n at
// cond + n cond_stride).  g_z[:C] = ga tanh(z_b) s (1 - s), g_z[C:] = ga s (1 - tanh(z_b)^2), s = sigmoid(z_a), into
// columns [layer 2 C, (layer + 1) 2 C) of gz [N, zcols] (fp32 and operand halves).  One thread per (token, channel).
__global__ void __launch_bounds__(256) df_gate_bwd_kernel(const float* __restrict__ ga, const float* __restrict__ g,
                                                          const float* __restrict__ cond, int cond_stride, int C,
                                                          int zcols, int layer, size_t n, float* __restrict__ gz,
                                                          float* __restrict__ gz_hi, float* __restrict__ gz_lo) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t tok = i / C;
        const int c = (int)(i - tok * C);
        const float* crow = cond + tok * cond_stride;
        const float za = g[tok * 2 * C + c] + crow[c], zb = g[tok * 2 * C + C + c] + crow[C + c];
        const float s = 1.0f / (1.0f + expf(-za)), th = tanhf(zb), gv = ga[i];
        const float ra = gv * th * (s * (1.0f - s)), rb = gv * s * (1.0f - th * th);
        const size_t k = tok * zcols + (size_t)layer * 2 * C + c;
        gz[k] = ra;
        gz[k + C] = rb;
        dfb_emit(ra, gz_hi, gz_lo, k);
        dfb_emit(rb, gz_hi, gz_lo, k + C);
    }
}

// One layer of the backward after its g_U GEMM.  gu [B T, 3 C] (NULL: the start, before the last layer, where h_L feeds
// nothing: gh = 0); gh [B T, C] in / out: the cotangent of h_{i+1} in, of h_i out = gh / sqrt 2 + g_y with
// g_y(t) = gu[t + 1, block 0] + gu[t, block 1] + gu[t - 1, block 2] inside utterance b (the adjoint of df_layer's
// scatter).  gr [B T, 2 C] (NULL after layer 0): [gh_out / sqrt 2 | gsk / skip_div], fp32 and operand halves.  part:
// the slab sums of g_y into column block `layer` of rf_layer_backward's layout (b n_slabs + s) (n_layers C) + layer C + c.
__global__ void __launch_bounds__(256) df_layer_bwd_kernel(const float* __restrict__ gu, float* __restrict__ gh,
                                                           const float* __restrict__ gsk, float skip_div, int T, int C,
                                                           int LC, int layer, int n_slabs, int n_items,
                                                           float* __restrict__ gr, float* __restrict__ gr_hi,
                                                           float* __restrict__ gr_lo, double* __restrict__ part) {
    const float kSqrt2 = 1.41421356237309515f;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int b = item / n_slabs, s = item - b * n_slabs;
        const int t0 = s * kDfSlab, t1 = min(t0 + kDfSlab, T);
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
            double acc = 0.0;
            for (int t = t0; t < t1; ++t) {
                const size_t n = (size_t)b * T + t, i = n * C + c;
                float h = 0.f;
                if (gu) {
                    const size_t r = n * 3 * C + c;
                    float gy = gu[r + C];
                    if (t + 1 < T) gy = gy + gu[r + 3 * C];                         // row t + 1, block 0
                    if (t > 0) gy = gy + gu[r - 3 * C + 2 * C];                     // row t - 1, block 2
                    h = __fadd_rn(gh[i] / kSqrt2, gy);
                    acc += (double)gy;
                }
                gh[i] = h;
                if (gr) {
                    const size_t k = n * 2 * C + c;
                    const float a = h / kSqrt2, sk = gsk[i] / skip_div;
                    gr[k] = a;
                    gr[k + C] = sk;
                    dfb_emit(a, gr_hi, gr_lo, k);
                    dfb_emit(sk, gr_hi, gr_lo, k + C);
                }
            }
            if (gu) part[(size_t)item * LC + (size_t)layer * C + c] = acc;
        }
    }
}

}  // namespace

#ifndef B2D_HOST_EMU
namespace {
unsigned dfb_grid(size_t work) {
    size_t g = (work + 255) / 256;
    const size_t cap = (size_t)b2d::num_sms() * 8;
    return (unsigned)(g < 1 ? 1 : g > cap ? cap : g);
}
int dfb_slabs(int T) { return (T + kDfSlab - 1) / kDfSlab; }
}  // namespace

extern "C" int b2d_df_loss_input(const float* gt, const float* noise, const int64_t* t, const float* sqrt_ac,
                                 const float* sqrt_1m_ac, int n_steps, float spec_min, float spec_range, int B, int T, int M,
                                 float* hi, float* lo, void* stream) {
    if (!gt || !noise || !t || !sqrt_ac || !sqrt_1m_ac || !hi) return b2d::fail(B2D_ERR_NULL, "df_loss_input: null pointer");
    if (B <= 0 || T <= 0 || M <= 0 || n_steps <= 0) return b2d::fail(B2D_ERR_SHAPE, "df_loss_input: bad shape");
    const size_t n = (size_t)B * T * M;
    df_loss_input_kernel<<<dfb_grid(n), 256, 0, (cudaStream_t)stream>>>(gt, noise, reinterpret_cast<const long long*>(t),
                                                                        sqrt_ac, sqrt_1m_ac, n_steps, spec_min, spec_range,
                                                                        T, M, n, hi, lo);
    return b2d::check_launch("df_loss_input");
}

extern "C" int b2d_df_relu_backward(const float* gy, const float* pre, const float* bias, int n_rows, int C, float* gx,
                                    float* hi, float* lo, void* stream) {
    if (!gy || !pre || !bias || !gx || (lo && !hi)) return b2d::fail(B2D_ERR_NULL, "df_relu_backward: null pointer");
    if (n_rows <= 0 || C <= 0) return b2d::fail(B2D_ERR_SHAPE, "df_relu_backward: bad shape");
    const size_t n = (size_t)n_rows * C;
    df_relu_bwd_kernel<<<dfb_grid(n), 256, 0, (cudaStream_t)stream>>>(gy, pre, bias, C, n, gx, hi, lo);
    return b2d::check_launch("df_relu_backward");
}

extern "C" int b2d_df_mish_backward(const float* gy, const float* x, int n, float* gx, float* hi, float* lo, void* stream) {
    if (!gy || !x || !gx || (lo && !hi)) return b2d::fail(B2D_ERR_NULL, "df_mish_backward: null pointer");
    if (n <= 0) return b2d::fail(B2D_ERR_SHAPE, "df_mish_backward: bad shape");
    df_mish_bwd_kernel<<<dfb_grid((size_t)n), 256, 0, (cudaStream_t)stream>>>(gy, x, (size_t)n, gx, hi, lo);
    return b2d::check_launch("df_mish_backward");
}

extern "C" int b2d_df_gate_backward(const float* ga, const float* g, const float* cond, int cond_stride, int n_tokens, int C,
                                    int layer, int n_layers, float* gz, float* gz_hi, float* gz_lo, void* stream) {
    if (!ga || !g || !cond || !gz || (gz_lo && !gz_hi)) return b2d::fail(B2D_ERR_NULL, "df_gate_backward: null pointer");
    if (n_tokens <= 0 || C <= 0 || cond_stride < 2 * C || n_layers <= 0 || layer < 0 || layer >= n_layers ||
        (long long)2 * C * n_layers > 0x7fffffffLL)
        return b2d::fail(B2D_ERR_SHAPE, "df_gate_backward: bad shape");
    const size_t n = (size_t)n_tokens * C;
    df_gate_bwd_kernel<<<dfb_grid(n), 256, 0, (cudaStream_t)stream>>>(ga, g, cond, cond_stride, C, 2 * C * n_layers, layer, n,
                                                                      gz, gz_hi, gz_lo);
    return b2d::check_launch("df_gate_backward");
}

extern "C" int b2d_df_layer_backward(const float* gu, float* gh, const float* gsk, float skip_div, int B, int T, int C,
                                     int layer, int n_layers, float* gr, float* gr_hi, float* gr_lo, void* ws,
                                     size_t ws_bytes, void* stream) {
    if (!gh || (gr && !gsk) || (gu && !ws) || (gr_hi && !gr) || (gr_lo && !gr_hi))
        return b2d::fail(B2D_ERR_NULL, "df_layer_backward: null pointer");
    if (B <= 0 || T <= 0 || C <= 0 || n_layers <= 0 || layer < 0 || layer >= n_layers || !(skip_div > 0.f) ||
        (long long)B * dfb_slabs(T) > 0x7fffffffLL || (long long)C * n_layers > 0x7fffffffLL)
        return b2d::fail(B2D_ERR_SHAPE, "df_layer_backward: bad shape");
    const int n_items = B * dfb_slabs(T);
    if (gu && ws_bytes < (size_t)n_items * C * n_layers * sizeof(double))
        return b2d::fail(B2D_ERR_WORKSPACE, "df_layer_backward: workspace too small");
    df_layer_bwd_kernel<<<dfb_grid((size_t)n_items * 256), 256, 0, (cudaStream_t)stream>>>(
        gu, gh, gsk, skip_div, T, C, C * n_layers, layer, dfb_slabs(T), n_items, gr, gr_hi, gr_lo, static_cast<double*>(ws));
    return b2d::check_launch("df_layer_backward");
}
#endif  // B2D_HOST_EMU
