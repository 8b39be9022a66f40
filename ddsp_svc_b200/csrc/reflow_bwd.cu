// The reflow model's training loss (reflow/reflow.py:20-35 and :63-68 with loss_type 'l2_lognorm') and the backward of
// the velocity network (reflow/naive_v2_diff.py:101-231 with conv_only, use_mlp=False).  The GEMMs and their adjoints
// (dX = gY W, dW = gY^T X), the GLU -> depthwise conv -> SiLU backward (unit2control_bwd.cu) and the bias column sums
// are issued by the host side (ddsp_svc_b200/reflow.py); these kernels are everything between them:
//
//   rf_loss_input     x_1 = norm(gt), x_t = x_0 + t_b (x_1 - x_0), target = x_1 - x_0 (x_0 token-major, t per utterance)
//   rf_loss           v = G + b_out, per-slab fp64 sums of w_b (target - v)^2, then the mean
//   rf_loss_backward  g_v = g_L 2 w_b (v - target) / (B M T)
//   rf_gelu_backward  g (Phi(x) + x phi(x)) of the exact-erf GELU (input projection, step MLP)
//   rf_layer_backward g_h += g_z of one layer; g_z into column block `layer` of G_Z; per-slab sums of g_z per utterance
//   rf_step_sums      the slabs of rf_layer_backward added per utterance: the step projection's cotangent g_S [B, L D]
//
// Activations are token-major [B, T, C] fp32.  Every output that feeds a GEMM is written as its operand: fp32, plus the
// TF32 (hi, lo) halves of a 3xTF32 product when the caller asks for them.  No atomics and no shared memory.  Sums over
// tokens are two-stage: a slab is a FIXED run of kSlab frames of one utterance, summed in frame order in fp64 by one
// thread per column; a second kernel adds the slabs in slab order in fp64.  The loops stride over slabs and columns by
// the launch's grid and block, so results do not depend on either and are bit-identical from run to run.
#ifndef B2D_HOST_EMU               // tests/emu/ runs these kernels' source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif
#include "tf32_split.cuh"
#include "token_slab.cuh"

namespace {

constexpr int kRfSlab = kTokenSlab;      // frames of one utterance per slab of a token sum

__device__ __forceinline__ void rfb_emit(float v, float* __restrict__ hi, float* __restrict__ lo, size_t i) {
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

// one thread per element of [B T, M]; x_t and target keep the reference's fp32 association (no contraction)
__global__ void __launch_bounds__(256) rf_loss_input_kernel(const float* __restrict__ gt, const float* __restrict__ x0,
                                                            const float* __restrict__ t, float spec_min, float spec_range,
                                                            int T, int M, size_t n, float* __restrict__ target,
                                                            float* __restrict__ hi, float* __restrict__ lo) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t b = i / ((size_t)T * M);
        const float x1 = ((gt[i] - spec_min) / spec_range) * 2.0f - 1.0f;          // reflow.py:107-108
        const float a = x0[i], d = __fsub_rn(x1, a);                               // reflow.py:22
        target[i] = d;
        rfb_emit(__fadd_rn(a, __fmul_rn(__ldg(t + b), d)), hi, lo, i);
    }
}

// part[(b n_slabs + s) M + m] = sum over the slab's frames of w_b ((target - v)^2), v = G + bias (fp64 sum of fp32 terms)
__global__ void __launch_bounds__(256) rf_loss_slabs_kernel(const float* __restrict__ g, const float* __restrict__ bias,
                                                            const float* __restrict__ target, const float* __restrict__ w,
                                                            int T, int M, int n_slabs, int n_items,
                                                            double* __restrict__ part) {
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int b = item / n_slabs, s = item - b * n_slabs;
        const int t0 = s * kRfSlab, t1 = min(t0 + kRfSlab, T);
        const float wb = __ldg(w + b);
        for (int m = threadIdx.x; m < M; m += blockDim.x) {
            const float bm = __ldg(bias + m);
            double acc = 0.0;
            for (int t = t0; t < t1; ++t) {
                const size_t i = ((size_t)b * T + t) * M + m;
                const float e = __fsub_rn(target[i], __fadd_rn(g[i], bm));
                acc += (double)__fmul_rn(wb, __fmul_rn(e, e));
            }
            part[(size_t)item * M + m] = acc;
        }
    }
}

// out[r n + j] = sum over s < n_slabs (in order, fp64) of part[(r n_slabs + s) n + j]; out_f32 or out_f64
__global__ void __launch_bounds__(256) rf_slab_reduce_kernel(const double* __restrict__ part, int n_rows, int n_slabs, int n,
                                                             float* __restrict__ out_f32, double* __restrict__ out_f64) {
    const size_t total = (size_t)n_rows * n;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (size_t)gridDim.x * blockDim.x) {
        const size_t r = e / n, j = e - r * n;
        const double* p = part + r * n_slabs * (size_t)n + j;
        double s = 0.0;
        for (int k = 0; k < n_slabs; ++k) s += p[(size_t)k * n];
        if (out_f32) out_f32[e] = (float)s;
        if (out_f64) out_f64[e] = s;
    }
}

// one thread: loss = (sum of the M column sums in order) / count
__global__ void rf_loss_finish_kernel(const double* __restrict__ cols, int M, double count, float* __restrict__ loss) {
    if (blockIdx.x != 0 || threadIdx.x != 0) return;
    double s = 0.0;
    for (int m = 0; m < M; ++m) s += cols[m];
    loss[0] = (float)(s / count);
}

// g_v = (g_L 2 w_b / count) (v - target), v = G + bias; fp32 into gv, operand halves into hi / lo (optional)
__global__ void __launch_bounds__(256) rf_loss_bwd_kernel(const float* __restrict__ g, const float* __restrict__ bias,
                                                          const float* __restrict__ target, const float* __restrict__ w,
                                                          const float* __restrict__ g_loss, double inv_count, int T, int M,
                                                          size_t n, float* __restrict__ gv, float* __restrict__ hi,
                                                          float* __restrict__ lo) {
    const double gl = (double)__ldg(g_loss) * 2.0 * inv_count;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t tok = i / M;
        const int m = (int)(i - tok * M);
        const float c = (float)(gl * (double)__ldg(w + tok / T));
        const float v = __fadd_rn(g[i], __ldg(bias + m));
        const float r = c * __fsub_rn(v, target[i]);
        gv[i] = r;
        rfb_emit(r, hi, lo, i);
    }
}

// gx = gy (Phi(x) + x phi(x)), x = pre (+ bias[c]) with the forward's association (rf_layer_input: G + b)
__global__ void __launch_bounds__(256) rf_gelu_bwd_kernel(const float* __restrict__ gy, const float* __restrict__ pre,
                                                          const float* __restrict__ bias, int C, size_t n,
                                                          float* __restrict__ gx, float* __restrict__ hi,
                                                          float* __restrict__ lo) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float x = bias ? __fadd_rn(pre[i], __ldg(bias + (int)(i % C))) : pre[i];
        const float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752f));
        const float pdf = 0.39894228040143268f * expf(-0.5f * x * x);
        const float r = gy[i] * (cdf + x * pdf);
        gx[i] = r;
        rfb_emit(r, hi, lo, i);
    }
}

// One layer of the backward after its g_z GEMM.  gz, gh [B T, D]; the residual stream's cotangent gh += gz in place, with
// its operand halves into gh_hi / gh_lo (optional); gz into column block `layer` of Z [B T, LD] (fp32 and halves); the
// slab sums of gz into part[(b n_slabs + s) LD + layer D + c] (fp64)
__global__ void __launch_bounds__(256) rf_layer_bwd_kernel(const float* __restrict__ gz, float* __restrict__ gh, int T, int D,
                                                           int LD, int layer, int n_slabs, int n_items,
                                                           float* __restrict__ gh_hi, float* __restrict__ gh_lo,
                                                           float* __restrict__ z, float* __restrict__ z_hi,
                                                           float* __restrict__ z_lo, double* __restrict__ part) {
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
        const int b = item / n_slabs, s = item - b * n_slabs;
        const int t0 = s * kRfSlab, t1 = min(t0 + kRfSlab, T);
        for (int c = threadIdx.x; c < D; c += blockDim.x) {
            double acc = 0.0;
            for (int t = t0; t < t1; ++t) {
                const size_t n = (size_t)b * T + t, i = n * D + c, k = n * LD + (size_t)layer * D + c;
                const float v = gz[i], h = __fadd_rn(gh[i], v);
                gh[i] = h;
                rfb_emit(h, gh_hi, gh_lo, i);
                z[k] = v;
                rfb_emit(v, z_hi, z_lo, k);
                acc += (double)v;
            }
            part[(size_t)item * LD + (size_t)layer * D + c] = acc;
        }
    }
}

}  // namespace

#ifndef B2D_HOST_EMU
namespace {
unsigned rfb_grid(size_t work) {
    size_t g = (work + 255) / 256;
    const size_t cap = (size_t)b2d::num_sms() * 8;
    return (unsigned)(g < 1 ? 1 : g > cap ? cap : g);
}
int rfb_slabs(int T) { return (T + kRfSlab - 1) / kRfSlab; }
size_t rfb_ws(int B, int T, int cols) { return (size_t)B * rfb_slabs(T) * cols * sizeof(double); }
bool rfb_bad(int B, int T, int C) { return B <= 0 || T <= 0 || C <= 0 || (long long)B * rfb_slabs(T) > 0x7fffffffLL; }
}  // namespace

extern "C" size_t b2d_rf_backward_workspace_bytes(int B, int T, int cols) {
    if (rfb_bad(B, T, cols)) return 0;
    return b2d::align256(rfb_ws(B, T, cols) + (size_t)cols * sizeof(double));
}

extern "C" int b2d_rf_loss_input(const float* gt, const float* x0, const float* t, float spec_min, float spec_range, int B,
                                 int T, int M, float* target, float* hi, float* lo, void* stream) {
    if (!gt || !x0 || !t || !target || !hi) return b2d::fail(B2D_ERR_NULL, "rf_loss_input: null pointer");
    if (B <= 0 || T <= 0 || M <= 0) return b2d::fail(B2D_ERR_SHAPE, "rf_loss_input: bad shape");
    const size_t n = (size_t)B * T * M;
    rf_loss_input_kernel<<<rfb_grid(n), 256, 0, (cudaStream_t)stream>>>(gt, x0, t, spec_min, spec_range, T, M, n, target, hi, lo);
    return b2d::check_launch("rf_loss_input");
}

extern "C" int b2d_rf_loss(const float* g, const float* bias, const float* target, const float* w, int B, int T, int M,
                           void* ws, size_t ws_bytes, float* loss, void* stream) {
    if (!g || !bias || !target || !w || !ws || !loss) return b2d::fail(B2D_ERR_NULL, "rf_loss: null pointer");
    if (rfb_bad(B, T, M)) return b2d::fail(B2D_ERR_SHAPE, "rf_loss: bad shape");
    if (ws_bytes < rfb_ws(B, T, M) + (size_t)M * sizeof(double)) return b2d::fail(B2D_ERR_WORKSPACE, "rf_loss: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    double* part = static_cast<double*>(ws);
    double* cols = part + (size_t)B * rfb_slabs(T) * M;
    const int n_items = B * rfb_slabs(T);
    rf_loss_slabs_kernel<<<rfb_grid((size_t)n_items * 256), 128, 0, st>>>(g, bias, target, w, T, M, rfb_slabs(T), n_items, part);
    rf_slab_reduce_kernel<<<rfb_grid((size_t)M), 256, 0, st>>>(part, 1, n_items, M, nullptr, cols);
    rf_loss_finish_kernel<<<1, 32, 0, st>>>(cols, M, (double)B * T * M, loss);
    return b2d::check_launch("rf_loss");
}

extern "C" int b2d_rf_loss_backward(const float* g, const float* bias, const float* target, const float* w,
                                    const float* g_loss, int B, int T, int M, float* gv, float* hi, float* lo, void* stream) {
    if (!g || !bias || !target || !w || !g_loss || !gv || (lo && !hi)) return b2d::fail(B2D_ERR_NULL, "rf_loss_backward: null pointer");
    if (B <= 0 || T <= 0 || M <= 0) return b2d::fail(B2D_ERR_SHAPE, "rf_loss_backward: bad shape");
    const size_t n = (size_t)B * T * M;
    rf_loss_bwd_kernel<<<rfb_grid(n), 256, 0, (cudaStream_t)stream>>>(g, bias, target, w, g_loss, 1.0 / ((double)n), T, M, n,
                                                                        gv, hi, lo);
    return b2d::check_launch("rf_loss_backward");
}

extern "C" int b2d_rf_gelu_backward(const float* gy, const float* pre, const float* bias, int n_rows, int C, float* gx,
                                    float* hi, float* lo, void* stream) {
    if (!gy || !pre || !gx || (lo && !hi)) return b2d::fail(B2D_ERR_NULL, "rf_gelu_backward: null pointer");
    if (n_rows <= 0 || C <= 0) return b2d::fail(B2D_ERR_SHAPE, "rf_gelu_backward: bad shape");
    const size_t n = (size_t)n_rows * C;
    rf_gelu_bwd_kernel<<<rfb_grid(n), 256, 0, (cudaStream_t)stream>>>(gy, pre, bias, C, n, gx, hi, lo);
    return b2d::check_launch("rf_gelu_backward");
}

extern "C" int b2d_rf_layer_backward(const float* gz, float* gh, int B, int T, int D, int layer, int n_layers, float* gh_hi,
                                     float* gh_lo, float* z, float* z_hi, float* z_lo, void* ws, size_t ws_bytes,
                                     void* stream) {
    if (!gz || !gh || !z || !ws || (gh_lo && !gh_hi) || (z_lo && !z_hi)) return b2d::fail(B2D_ERR_NULL, "rf_layer_backward: null pointer");
    if (rfb_bad(B, T, D) || n_layers <= 0 || layer < 0 || layer >= n_layers || (long long)D * n_layers > 0x7fffffffLL)
        return b2d::fail(B2D_ERR_SHAPE, "rf_layer_backward: bad shape");
    if (ws_bytes < rfb_ws(B, T, D * n_layers)) return b2d::fail(B2D_ERR_WORKSPACE, "rf_layer_backward: workspace too small");
    const int n_items = B * rfb_slabs(T);
    rf_layer_bwd_kernel<<<rfb_grid((size_t)n_items * 256), 256, 0, (cudaStream_t)stream>>>(
        gz, gh, T, D, D * n_layers, layer, rfb_slabs(T), n_items, gh_hi, gh_lo, z, z_hi, z_lo, static_cast<double*>(ws));
    return b2d::check_launch("rf_layer_backward");
}

extern "C" int b2d_rf_step_sums(const void* ws, size_t ws_bytes, int B, int T, int cols, float* out, void* stream) {
    if (!ws || !out) return b2d::fail(B2D_ERR_NULL, "rf_step_sums: null pointer");
    if (rfb_bad(B, T, cols)) return b2d::fail(B2D_ERR_SHAPE, "rf_step_sums: bad shape");
    if (ws_bytes < rfb_ws(B, T, cols)) return b2d::fail(B2D_ERR_WORKSPACE, "rf_step_sums: workspace too small");
    rf_slab_reduce_kernel<<<rfb_grid((size_t)B * cols), 256, 0, (cudaStream_t)stream>>>(static_cast<const double*>(ws), B,
                                                                                      rfb_slabs(T), cols, out, nullptr);
    return b2d::check_launch("rf_step_sums");
}
#endif  // B2D_HOST_EMU
