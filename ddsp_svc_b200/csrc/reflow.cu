// Fused stages of the reflow model's rectified-flow sampler (reflow/reflow.py:51-105 around the velocity network
// reflow/naive_v2_diff.py:101-231 with conv_only, use_mlp=False).  The velocity network's products (input projection,
// each layer's two pointwise convolutions, output projection) are library GEMMs issued by the host side
// (ddsp_svc_b200/reflow.py) and its GLU -> depthwise conv -> SiLU stage is unit2control.cu's; these kernels are everything
// between those GEMMs:
//
//   rf_start        x0 = t_start norm(gt) + (1 - t_start) noise, the noise read channel-major [B, 1, M, T]
//   rf_layer_input  h = GELU(G + b) (input projection) or h = (G + b) + h (a layer's residual), then the next layer's
//                   input h + S[b] + C[b, t] (step and condition projections), or h itself after the last layer
//   rf_ode_update   v = G + b_out; Euler x += v dt, or one RK4 stage (k1 + 2 k2 + 2 k3 + k4 accumulator)
//   rf_finish       denorm(x) into the [B, T, M] output
//
// Activations are token-major [B, T, C] fp32.  Every kernel that feeds a GEMM writes the GEMM's operand: fp32 (lo NULL)
// or the TF32 (hi, lo) halves of a 3xTF32 product, so no separate split pass runs.  All are elementwise (one owner per
// output element, no atomics, no reductions): results are bit-identical from run to run.  The expressions keep the
// reference's fp32 association so the sampler's own rounding matches the reference's.
#ifndef B2D_HOST_EMU               // tests/emu/ runs these kernels' source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif
#include "tf32_split.cuh"

namespace {

__device__ __forceinline__ void rf_emit(float v, float* __restrict__ hi, float* __restrict__ lo, size_t i) {
    if (lo) {
        float h, l;
        tf32_split(v, h, l);
        hi[i] = h;
        lo[i] = l;
    } else {
        hi[i] = v;
    }
}

// exact-erf GELU with torch's association: x * 0.5 * (1 + erf(x / sqrt 2))
__device__ __forceinline__ float rf_gelu(float x) { return (x * 0.5f) * (1.0f + erff(x * 0.70710678118654752f)); }

// one thread per element of x [n_tokens, M], m fastest (coalesced writes; the transposed noise read is once per call)
__global__ void __launch_bounds__(256) rf_start_kernel(const float* __restrict__ noise, const float* __restrict__ gt,
                                                       float t_start, float one_minus_t_start, float spec_min,
                                                       float spec_range, int T, int M, size_t n, float* __restrict__ x,
                                                       float* __restrict__ hi, float* __restrict__ lo) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const size_t tok = i / M;
        const int m = (int)(i - tok * M);
        const size_t b = tok / T;
        const int t = (int)(tok - b * T);
        float v = noise[(b * M + m) * T + t];
        if (gt) {
            const float nrm = ((gt[i] - spec_min) / spec_range) * 2.0f - 1.0f;         // reflow.py:107-108
            v = t_start * nrm + one_minus_t_start * v;
        }
        if (x) x[i] = v;
        rf_emit(v, hi, lo, i);
    }
}

// G, h [n_tokens, D]; step: row b at step + b * step_stride; cond: row n at cond + n * cond_stride (both NULL after the
// last layer).  One thread per 4 channels.
__global__ void __launch_bounds__(256) rf_layer_input_kernel(const float4* __restrict__ g, const float4* __restrict__ bias,
                                                             float4* __restrict__ h, int residual,
                                                             const float* __restrict__ step, int step_stride,
                                                             const float* __restrict__ cond, int cond_stride, int T,
                                                             int D4, size_t n4, float* __restrict__ hi,
                                                             float* __restrict__ lo) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        const size_t tok = i / D4;
        const int c4 = (int)(i - tok * D4);
        const float4 gv = g[i], bv = __ldg(bias + c4);
        float r[4] = {gv.x + bv.x, gv.y + bv.y, gv.z + bv.z, gv.w + bv.w};
        if (residual) {                      // naive_v2_diff.py:94-96: conformer(x) + res_x
            const float4 hv = h[i];
            r[0] = r[0] + hv.x; r[1] = r[1] + hv.y; r[2] = r[2] + hv.z; r[3] = r[3] + hv.w;
        } else {                             // naive_v2_diff.py:209-210: gelu(input_projection(x))
            for (int k = 0; k < 4; ++k) r[k] = rf_gelu(r[k]);
        }
        h[i] = make_float4(r[0], r[1], r[2], r[3]);
        if (step) {                          // naive_v2_diff.py:83: x + diffusion_step_projection + condition_projection
            const float4 sv = *reinterpret_cast<const float4*>(step + (tok / T) * step_stride + 4 * c4);
            const float4 cv = *reinterpret_cast<const float4*>(cond + tok * cond_stride + 4 * c4);
            r[0] = (r[0] + sv.x) + cv.x; r[1] = (r[1] + sv.y) + cv.y; r[2] = (r[2] + sv.z) + cv.z; r[3] = (r[3] + sv.w) + cv.w;
        }
        for (int k = 0; k < 4; ++k) rf_emit(r[k], hi, lo, 4 * i + k);
    }
}

// v = G + b_out.  stage < 0: Euler, x += v dt, emits x (reflow.py:37-40).  RK4 (reflow.py:42-49), emitting the next
// evaluation's input: stage 0: acc = v, emits x + (0.5 v) dt; 1: acc += 2 v, emits x + (0.5 v) dt; 2: acc += 2 v, emits
// x + v dt; 3: x += ((acc + v) dt) / 6, emits x.
__global__ void __launch_bounds__(256) rf_ode_kernel(const float* __restrict__ g, const float* __restrict__ bias,
                                                     float* __restrict__ x, float* __restrict__ acc, int stage, float dt,
                                                     int M, size_t n, float* __restrict__ hi, float* __restrict__ lo) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float v = g[i] + __ldg(bias + (int)(i % M));
        float xv = x[i], out;
        if (stage < 0) {
            xv = xv + v * dt;
            x[i] = xv;
            out = xv;
        } else if (stage == 3) {
            xv = xv + ((acc[i] + v) * dt) / 6.0f;
            x[i] = xv;
            out = xv;
        } else {
            acc[i] = stage == 0 ? v : acc[i] + 2.0f * v;
            out = xv + (stage == 2 ? v * dt : (0.5f * v) * dt);
        }
        rf_emit(out, hi, lo, i);
    }
}

// out = denorm(x) = ((x + 1) / 2) (spec_max - spec_min) + spec_min (reflow.py:110-111)
__global__ void __launch_bounds__(256) rf_finish_kernel(const float* __restrict__ x, float spec_min, float spec_range,
                                                        size_t n, float* __restrict__ out) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        out[i] = ((x[i] + 1.0f) / 2.0f) * spec_range + spec_min;
}

}  // namespace

#ifndef B2D_HOST_EMU
namespace {
unsigned rf_grid(size_t work) {
    size_t g = (work + 255) / 256;
    const size_t cap = (size_t)b2d::num_sms() * 8;
    return (unsigned)(g < 1 ? 1 : g > cap ? cap : g);
}
}  // namespace

extern "C" int b2d_rf_start(const float* noise, const float* gt, float t_start, float one_minus_t_start, float spec_min,
                            float spec_range, int B, int T, int M, float* x, float* hi, float* lo, void* stream) {
    if (!noise || !hi) return b2d::fail(B2D_ERR_NULL, "rf_start: null pointer");
    if (B <= 0 || T <= 0 || M <= 0) return b2d::fail(B2D_ERR_SHAPE, "rf_start: bad shape");
    const size_t n = (size_t)B * T * M;
    rf_start_kernel<<<rf_grid(n), 256, 0, (cudaStream_t)stream>>>(noise, gt, t_start, one_minus_t_start, spec_min, spec_range,
                                                                  T, M, n, x, hi, lo);
    return b2d::check_launch("rf_start");
}

extern "C" int b2d_rf_layer_input(const float* g, const float* bias, float* h, int residual, const float* step,
                                  int step_stride, const float* cond, int cond_stride, int B, int T, int D, float* hi,
                                  float* lo, void* stream) {
    if (!g || !bias || !h || !hi || (!step != !cond)) return b2d::fail(B2D_ERR_NULL, "rf_layer_input: null pointer");
    if (B <= 0 || T <= 0 || D <= 0 || (step && ((step_stride != 0 && step_stride < D) || cond_stride < D)))
        return b2d::fail(B2D_ERR_SHAPE, "rf_layer_input: bad shape");
    if (D % 4 || !b2d::aligned16(g) || !b2d::aligned16(bias) || !b2d::aligned16(h) ||
        (step && (step_stride % 4 || cond_stride % 4 || !b2d::aligned16(step) || !b2d::aligned16(cond))))
        return b2d::fail(B2D_ERR_ALIGN, "rf_layer_input: width, strides and buffers must be 16-byte multiples");
    const size_t n4 = (size_t)B * T * (D / 4);
    rf_layer_input_kernel<<<rf_grid(n4), 256, 0, (cudaStream_t)stream>>>(
        reinterpret_cast<const float4*>(g), reinterpret_cast<const float4*>(bias), reinterpret_cast<float4*>(h), residual,
        step, step_stride, cond, cond_stride, T, D / 4, n4, hi, lo);
    return b2d::check_launch("rf_layer_input");
}

extern "C" int b2d_rf_ode_update(const float* g, const float* bias, float* x, float* acc, int stage, float dt, int n_tokens,
                                 int M, float* hi, float* lo, void* stream) {
    if (!g || !bias || !x || !hi || (stage >= 0 && !acc)) return b2d::fail(B2D_ERR_NULL, "rf_ode_update: null pointer");
    if (n_tokens <= 0 || M <= 0) return b2d::fail(B2D_ERR_SHAPE, "rf_ode_update: bad shape");
    if (stage < -1 || stage > 3) return b2d::fail(B2D_ERR_UNSUPPORTED, "rf_ode_update: stage must be -1 (Euler) or 0..3 (RK4)");
    const size_t n = (size_t)n_tokens * M;
    rf_ode_kernel<<<rf_grid(n), 256, 0, (cudaStream_t)stream>>>(g, bias, x, acc, stage, dt, M, n, hi, lo);
    return b2d::check_launch("rf_ode_update");
}

extern "C" int b2d_rf_finish(const float* x, float spec_min, float spec_range, int n, float* out, void* stream) {
    if (!x || !out) return b2d::fail(B2D_ERR_NULL, "rf_finish: null pointer");
    if (n <= 0) return b2d::fail(B2D_ERR_SHAPE, "rf_finish: bad shape");
    rf_finish_kernel<<<rf_grid((size_t)n), 256, 0, (cudaStream_t)stream>>>(x, spec_min, spec_range, (size_t)n, out);
    return b2d::check_launch("rf_finish");
}
#endif  // B2D_HOST_EMU
