// Fused non-causal linear attention of the performer (FAVOR+) layers of PCmer -- reference ddsp/pcmer.py:220-229
// (`linear_attention`) on the feature maps q' = phi(q), k' = phi(k) of csrc/unit2control.cu:
//
//   k_sum   = sum_t k'[t, :]                      [J]
//   context = sum_t k'[t, :]^T v[t, :]            [J, D]
//   out[t]  = (q'[t, :] . context) / (q'[t, :] . k_sum + 1e-8)
//
// One CTA per (utterance, head).  The reference (and the first version of ddsp_svc_b200/unit2control.py) runs this as two
// batched GEMMs of 256 small problems plus three eager elementwise passes; here k_sum and context (J x D = 266 x 64 floats,
// 68 KB) are built once in shared memory while k' and v stream through in tiles of 16 frames, then q' streams through and
// every output row is finished (contraction, normaliser, division) in registers and written straight in the [B, T, H, D]
// layout the output projection reads -- q', k', v are read exactly once, nothing intermediate touches HBM.
//   phase A: 34 x 8 threads, each an 8 (features) x 8 (channels) register tile of context (+ k_sum on the first channel group)
//   phase B: 16 frames x 16 channel quads per tile: thread = (frame, 4 channels), J-long dot products against the shared context
// Logic pinned on the CPU by the host emulation (tests/test_emu_linear_attention.py) against the fp64 formula.
#ifndef B2D_HOST_EMU
#include "b2d_common.cuh"
#endif

namespace {

constexpr int kLaD = 64;                 // dim_head of the reference's SelfAttention (pcmer.py:313)
constexpr int kLaJmax = 272;             // features padded to a multiple of 8 (266 = int(64 ln 64))
constexpr int kLaTT = 16;                // frames per tile
constexpr int kLaThreads = 288;          // 272 compute threads of phase A (34 feature groups x 8 channel groups) + 16 loaders
// phase A sums 64 frames in registers, then adds them to the totals in shared memory: one fp32 chain over all T frames
// had 7x the error of the library path (kf.sum + fp32 GEMM) at T = 5168, J = 8; two chains of about sqrt(T) do not
constexpr int kLaFlushTiles = 4;

struct LinAttnParams {
    const float* qf;       // [BH, T, J]
    const float* kf;       // [BH, T, J]
    const float* v;        // [BH, T, D]
    float* out;            // [B, T, H, D]
    int T, J, H;
    float eps;
};

constexpr size_t kLaSmemFloats = (size_t)kLaJmax * kLaD + kLaJmax + (size_t)kLaTT * kLaJmax + (size_t)kLaTT * kLaD;

__global__ void __launch_bounds__(kLaThreads, 2) u2c_linear_attention_kernel(LinAttnParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* ctx = reinterpret_cast<float*>(smem_raw);        // [kLaJmax][64]
    float* ksum = ctx + kLaJmax * kLaD;                     // [kLaJmax]
    float* ftile = ksum + kLaJmax;                          // [16][kLaJmax]  k' tile (phase A) / q' tile (phase B)
    float* vtile = ftile + kLaTT * kLaJmax;                 // [16][64]
    const int tid = threadIdx.x, bh = blockIdx.x;
    const int T = p.T, J = p.J;
    const float* kf = p.kf + (size_t)bh * T * J;
    const float* qf = p.qf + (size_t)bh * T * J;
    const float* v = p.v + (size_t)bh * T * kLaD;

    // ---- phase A: context and k_sum ----
    const int jg = tid >> 3, dg = tid & 7;                  // tid < 272: features 8 jg .. 8 jg + 7, channels 8 dg .. 8 dg + 7
    float acc[8][8], ks[8];
#pragma unroll
    for (int a = 0; a < 8; ++a) {
        ks[a] = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[a][c] = 0.f;
    }
    if (tid < 272) {                                        // each thread owns its 8 x 8 block of the totals
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
            for (int k = 0; k < 8; ++k) ctx[(8 * jg + i) * kLaD + 8 * dg + k] = 0.f;
            if (dg == 0) ksum[8 * jg + i] = 0.f;
        }
    }
    for (int t0 = 0, tile = 1; t0 < T; t0 += kLaTT, ++tile) {
        for (int i = tid; i < kLaTT * kLaJmax; i += kLaThreads) {
            const int tt = i / kLaJmax, j = i - tt * kLaJmax;
            ftile[i] = (t0 + tt < T && j < J) ? kf[(size_t)(t0 + tt) * J + j] : 0.f;
        }
        for (int i = tid; i < kLaTT * kLaD; i += kLaThreads) {
            const int tt = i / kLaD;
            vtile[i] = (t0 + tt < T) ? v[(size_t)(t0 + tt) * kLaD + (i - tt * kLaD)] : 0.f;
        }
        __syncthreads();
        if (tid < 272) {
#pragma unroll 4
            for (int tt = 0; tt < kLaTT; ++tt) {
                float a[8], c[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) { a[i] = ftile[tt * kLaJmax + 8 * jg + i]; c[i] = vtile[tt * kLaD + 8 * dg + i]; }
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    ks[i] += a[i];
#pragma unroll
                    for (int k = 0; k < 8; ++k) acc[i][k] = fmaf(a[i], c[k], acc[i][k]);
                }
            }
            if (tile % kLaFlushTiles == 0 || t0 + kLaTT >= T) {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
#pragma unroll
                    for (int k = 0; k < 8; ++k) { ctx[(8 * jg + i) * kLaD + 8 * dg + k] += acc[i][k]; acc[i][k] = 0.f; }
                    if (dg == 0) ksum[8 * jg + i] += ks[i];
                    ks[i] = 0.f;
                }
            }
        }
        __syncthreads();
    }

    // ---- phase B: out[t] = (q'[t] . context) / (q'[t] . k_sum + eps) ----
    const int b = bh / p.H, h = bh - b * p.H;
    const int tt_b = tid >> 4, dq = tid & 15;               // tid < 256: frame tt_b of the tile, channels 4 dq .. 4 dq + 3
    for (int t0 = 0; t0 < T; t0 += kLaTT) {
        for (int i = tid; i < kLaTT * kLaJmax; i += kLaThreads) {
            const int tt = i / kLaJmax, j = i - tt * kLaJmax;
            ftile[i] = (t0 + tt < T && j < J) ? qf[(size_t)(t0 + tt) * J + j] : 0.f;
        }
        __syncthreads();
        if (tid < 256 && t0 + tt_b < T) {
            float n0 = 0.f, n1 = 0.f, n2 = 0.f, n3 = 0.f, den = 0.f;
            const float* qrow = ftile + tt_b * kLaJmax;
#pragma unroll 2
            for (int j = 0; j < J; ++j) {
                const float qv = qrow[j];
                const float* cr = ctx + j * kLaD + 4 * dq;
                n0 = fmaf(qv, cr[0], n0); n1 = fmaf(qv, cr[1], n1); n2 = fmaf(qv, cr[2], n2); n3 = fmaf(qv, cr[3], n3);
                den = fmaf(qv, ksum[j], den);
            }
            const float dinv = 1.0f / (den + p.eps);
            float* o = p.out + (((size_t)b * T + (t0 + tt_b)) * p.H + h) * kLaD + 4 * dq;
            o[0] = n0 * dinv; o[1] = n1 * dinv; o[2] = n2 * dinv; o[3] = n3 * dinv;
        }
        __syncthreads();
    }
}

}  // namespace

#ifndef B2D_HOST_EMU
extern "C" int b2d_u2c_linear_attention(const float* q_features, const float* k_features, const float* v, float* out, int B,
                                        int H, int T, int n_features, int dim_head, float eps, void* stream) {
    if (!q_features || !k_features || !v || !out) return b2d::fail(B2D_ERR_NULL, "u2c_linear_attention: null pointer");
    if (B <= 0 || H <= 0 || T <= 0 || n_features <= 0) return b2d::fail(B2D_ERR_SHAPE, "u2c_linear_attention: bad shape");
    if (dim_head != kLaD || n_features > kLaJmax)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "u2c_linear_attention: built for dim_head %d and at most %d features (got %d, %d)", kLaD,
                         kLaJmax, dim_head, n_features);
    LinAttnParams p;
    p.qf = q_features; p.kf = k_features; p.v = v; p.out = out; p.T = T; p.J = n_features; p.H = H; p.eps = eps;
    const size_t smem = kLaSmemFloats * sizeof(float);
    cudaError_t e = cudaFuncSetAttribute(u2c_linear_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return b2d::fail((int)e, "u2c_linear_attention: smem attr: %s", cudaGetErrorString(e));
    u2c_linear_attention_kernel<<<(unsigned)(B * H), kLaThreads, smem, (cudaStream_t)stream>>>(p);
    return b2d::check_launch("u2c_linear_attention");
}
#endif
