// Backward of the performer self-attention of the PCmer decoder (Unit2Control without use_naive_v2: ddsp/pcmer.py:14-47,
// :220-229, :283-309, :343-381): the elementwise and row-reduction stages between the library GEMMs that the host side
// (ddsp_svc_b200/unit2control.py) issues.  Rows are (utterance b, head h, frame t); one warp owns one row:
//
//   u2c_attn_readout_bwd  out = (phi_q ctx) / D with D = phi_q . ksum + 1e-8  ->  [g_num | g_D], 65 columns head-major,
//                         so ONE batched product phi_q^T [g_num | g_D] gives g_ctx and g_ksum together
//   u2c_feat_bwd          adjoint of the softmax-kernel feature map (+ the rank-1 terms of the read-out the GEMMs leave out):
//                         g_dd in place of g_phi, and the diag term of g_data (the host adds g_dd proj onto it)
//   u2c_qkv_gather_bwd    head-major g_q, g_k, g_v -> token-major g_qkv [N, 3 H 64] for the packed qkv GEMMs, with the
//                         pcmer_norm adjoint of q / (|q| + 1e-8) fused in
//
// No atomics and no shared memory: every output element has one owning warp and every sum runs over one row in a fixed
// butterfly order, so results are bit-identical from run to run.  A warp past the last row still joins the shuffles (the
// row index is clamped) and only skips its stores: every warp of a CTA runs the same shuffle sequence.
#ifndef B2D_HOST_EMU               // tests/emu/ runs this source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif

namespace {

constexpr int kHd = 64;            // dim_head: a row of q / k / v is two floats per lane
constexpr int kJmax = 288;         // n_features <= 9 per lane (the reference's int(64 ln 64) = 266)
constexpr int kJper = kJmax / 32;
constexpr int kRowsPerCta = 8;     // 256 threads

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    return v;
}

// g_out [B, T, H, 64] (token-major: the cotangent of the read-out before to_out) and out (the forward's read-out, same
// layout), d_inv [B, H, T] = 1 / D  ->  gn [B, H, T, 65]: g_num = g_out / D, then g_D = -(g_out . out) / D
__global__ void __launch_bounds__(256) u2c_attn_readout_bwd_kernel(const float* __restrict__ g_out, const float* __restrict__ out,
                                                                   const float* __restrict__ d_inv, int H, int T, int rows,
                                                                   float* __restrict__ gn) {
    const int lane = threadIdx.x & 31, row = blockIdx.x * kRowsPerCta + (threadIdx.x >> 5);
    const int r = min(row, rows - 1);
    const int t = r % T, bh = r / T, h = bh % H, b = bh / H;
    const size_t tok = (((size_t)b * T + t) * H + h) * kHd;
    const float di = d_inv[r];
    const float g0 = g_out[tok + lane], g1 = g_out[tok + 32 + lane];
    const float dot = warp_sum(fmaf(g1, out[tok + 32 + lane], g0 * out[tok + lane]));
    if (row >= rows) return;
    float* o = gn + (size_t)r * (kHd + 1);
    o[lane] = g0 * di;
    o[32 + lane] = g1 * di;
    if (lane == 0) o[kHd] = -dot * di;
}

// Feature map of one row (x = data row, dd = x (d^-1/4 proj)^T, r = J^-1/2, diag = |x|^2 / 2 d^-1/2):
//   query  phi_j = r (exp(dd_j - diag - max_j dd) + eps)    key  phi_j = r exp(dd_j - diag + eps)
// With the full feature cotangent gf_j = g_j + scal vec_j (query: g_D ksum_j; key: g_ksum_j) and
// ga_j = gf_j d phi_j / d dd_j (query: r E_j = phi_j - r eps; key: phi_j), s = sum_j ga_j:
//   g_dd_j = ga_j (- s at the row's maximum, queries: the reference's max is not detached);  g_x = -s d^-1/2 x
// The maximum's index is the first maximum of the saved phi row (phi is increasing in dd).  phi_j - r eps cancels where
// E_j << eps; its absolute error stays below |gf_j| r eps 2^-24.
__global__ void __launch_bounds__(256) u2c_feat_bwd_kernel(float* __restrict__ g, const float* __restrict__ phi,
                                                           const float* __restrict__ data, const float* __restrict__ vec,
                                                           const float* __restrict__ scal, int rows, int T, int J, int is_query,
                                                           float eps, float* __restrict__ gx) {
    const int lane = threadIdx.x & 31, row = blockIdx.x * kRowsPerCta + (threadIdx.x >> 5);
    const int r = min(row, rows - 1);
    const float ratio = rsqrtf((float)J), reps = ratio * eps;
    const float sc = scal ? scal[r] : 1.0f;
    const float* pr = phi + (size_t)r * J;
    const float* vr = vec + (size_t)(r / T) * J;
    float* gr = g + (size_t)r * J;
    float ga[kJper], s = 0.f, best = -INFINITY;
    int bi = J;
#pragma unroll
    for (int i = 0; i < kJper; ++i) {
        const int j = lane + 32 * i;
        float a = 0.f;
        if (j < J) {
            const float p = pr[j];
            a = fmaf(sc, vr[j], gr[j]) * (is_query ? p - reps : p);
            if (p > best) { best = p; bi = j; }
        }
        ga[i] = a;
        s += a;
    }
    s = warp_sum(s);
    if (is_query) {
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, d);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, d);
            if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
    }
    if (row >= rows) return;
#pragma unroll
    for (int i = 0; i < kJper; ++i) {
        const int j = lane + 32 * i;
        if (j < J) gr[j] = (is_query && j == bi) ? ga[i] - s : ga[i];
    }
    const float c = -s * (1.0f / 8.0f);                  // d^-1/2 at d = 64, as the forward's (d^-1/4)^2
    const float* xr = data + (size_t)r * kHd;
    float* o = gx + (size_t)r * kHd;
    o[lane] = c * xr[lane];
    o[32 + lane] = c * xr[32 + lane];
}

// gq, gk, gv [B, H, T, 64] head-major -> gqkv [B, T, 3, H, 64] token-major (the packed to_q | to_k | to_v output).
// normalized (pcmer_norm): gq / gk are cotangents of x / (n + 1e-8), n = |x|, with x the raw projection read from qkv (the
// forward's GEMM output, gqkv's layout):  g_x = g / (n + e) - x (x . g) / (n (n + e)^2)   (0 for the second term at n = 0)
__global__ void __launch_bounds__(256) u2c_qkv_gather_bwd_kernel(const float* __restrict__ gq, const float* __restrict__ gk,
                                                                 const float* __restrict__ gv, const float* __restrict__ qkv, int H,
                                                                 int T, int rows, int normalized, float* __restrict__ gqkv) {
    const int lane = threadIdx.x & 31, row = blockIdx.x * kRowsPerCta + (threadIdx.x >> 5);
    const int r = min(row, rows - 1);
    const int t = r % T, bh = r / T, h = bh % H, b = bh / H;
    const size_t src = (size_t)r * kHd, dst = ((size_t)b * T + t) * 3 * H * kHd + (size_t)h * kHd;
#pragma unroll
    for (int which = 0; which < 3; ++which) {
        const float* gs = which == 0 ? gq : which == 1 ? gk : gv;
        float g0 = gs[src + lane], g1 = gs[src + 32 + lane];
        const size_t o = dst + (size_t)which * H * kHd;
        if (normalized && which < 2) {
            const float x0 = qkv[o + lane], x1 = qkv[o + 32 + lane];
            const float n = sqrtf(warp_sum(fmaf(x1, x1, x0 * x0)));
            const float xg = warp_sum(fmaf(x1, g1, x0 * g0));
            const float ne = n + 1e-8f, a = 1.0f / ne, c = n > 0.f ? xg / (n * ne * ne) : 0.f;
            g0 = fmaf(g0, a, -x0 * c);
            g1 = fmaf(g1, a, -x1 * c);
        }
        if (row < rows) {
            gqkv[o + lane] = g0;
            gqkv[o + 32 + lane] = g1;
        }
    }
}

}  // namespace

#ifndef B2D_HOST_EMU

namespace {
inline unsigned ctas(long long rows) { return (unsigned)((rows + kRowsPerCta - 1) / kRowsPerCta); }
}  // namespace

extern "C" int b2d_u2c_attn_readout_backward(const float* g_out, const float* out, const float* d_inv, int B, int H, int T,
                                             int dim_head, float* gn, void* stream) {
    if (!g_out || !out || !d_inv || !gn) return b2d::fail(B2D_ERR_NULL, "u2c_attn_readout_backward: null pointer");
    if (B <= 0 || H <= 0 || T <= 0 || dim_head != kHd || (long long)B * H * T > 0x7fffffffLL)
        return b2d::fail(B2D_ERR_SHAPE, "u2c_attn_readout_backward: needs dim_head = 64");
    const int rows = B * H * T;
    u2c_attn_readout_bwd_kernel<<<ctas(rows), 256, 0, (cudaStream_t)stream>>>(g_out, out, d_inv, H, T, rows, gn);
    return b2d::check_launch("u2c_attn_readout_backward");
}

extern "C" int b2d_u2c_softmax_features_backward(float* g, const float* features, const float* data, const float* vec,
                                                 const float* scal, int rows, int T, int n_features, int dim_head, int is_query,
                                                 float eps, float* gx, void* stream) {
    if (!g || !features || !data || !vec || !gx || (is_query && !scal))
        return b2d::fail(B2D_ERR_NULL, "u2c_softmax_features_backward: null pointer");
    if (rows <= 0 || T <= 0 || rows % T || n_features <= 0 || n_features > kJmax || dim_head != kHd)
        return b2d::fail(B2D_ERR_SHAPE, "u2c_softmax_features_backward: needs dim_head = 64, n_features <= 288, rows a multiple of T");
    u2c_feat_bwd_kernel<<<ctas(rows), 256, 0, (cudaStream_t)stream>>>(g, features, data, vec, is_query ? scal : nullptr, rows, T,
                                                                       n_features, is_query ? 1 : 0, eps, gx);
    return b2d::check_launch("u2c_softmax_features_backward");
}

extern "C" int b2d_u2c_qkv_gather_backward(const float* gq, const float* gk, const float* gv, const float* qkv, int B, int H, int T,
                                           int dim_head, int normalized, float* gqkv, void* stream) {
    if (!gq || !gk || !gv || !gqkv || (normalized && !qkv)) return b2d::fail(B2D_ERR_NULL, "u2c_qkv_gather_backward: null pointer");
    if (B <= 0 || H <= 0 || T <= 0 || dim_head != kHd || (long long)B * H * T > 0x7fffffffLL)
        return b2d::fail(B2D_ERR_SHAPE, "u2c_qkv_gather_backward: needs dim_head = 64");
    const int rows = B * H * T;
    u2c_qkv_gather_bwd_kernel<<<ctas(rows), 256, 0, (cudaStream_t)stream>>>(gq, gk, gv, qkv, H, T, rows, normalized ? 1 : 0, gqkv);
    return b2d::check_launch("u2c_qkv_gather_backward");
}

#endif  // B2D_HOST_EMU
