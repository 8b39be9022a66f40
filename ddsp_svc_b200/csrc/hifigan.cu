// The NSF-HiFiGAN generator (nsf_hifigan/models.py:207-273), inference, as two kernels:
//
//   hg_conv  one dilated Conv1d as an implicit GEMM on the tensor cores (mma.sync m16n8k8 TF32, 3xTF32: both operands
//            split into TF32 (hi, lo), hi.hi + lo.hi + hi.lo per product).  Activations are token-major
//            [B, T, C] fp32.  A CTA owns BM time rows of one utterance x BN output channels; per 16-channel chunk of the
//            input it stages the BM rows plus a halo of d (k - 1) / 2 rows per side in shared memory once (cp.async,
//            double buffered; rows outside the utterance land as zeros) and takes all k taps from that tile, so no
//            im2col operand is ever written.  Prologue: leaky_relu(x, 0.1) or nothing.  Epilogue: + bias, then
//            + residual, + accum (the MRF sum) and / div, each optional -- a ResBlock1 is 6 launches and the last one of
//            a stage writes (xs + r) / num_kernels straight into the next stage's input.
//            The ConvTranspose1d(C_in, C_out, 2u, u, u / 2) of each stage runs through the same kernel in polyphase
//            form: a k = 3 convolution over input frames m - 1, m, m + 1 with u C_out outputs (column r C_out + co is
//            output phase r, its taps r + u / 2 + u, r + u / 2, r + u / 2 - u of the original kernel, the one outside
//            [0, 2u) zero; the host packs them).  Its epilogue interleaves the phases into [B, T u, C_out], adds the bias
//            and the stage's noise_convs[i](har_source) term, a strided dot of n_k taps over the [B, T_src] source.
//   hg_post  leaky_relu(x, 0.01) -> Conv1d(C -> 1, k 7, padding 3) -> tanh into [B, 1, T].
//
// Weights arrive split into TF32 (hi, lo) in the B-fragment order of mma.sync (weight-norm folded, see
// ddsp_svc_b200/hifigan.py): for tap j, the 8-channel block kb of the input and the 8-column block nb of the output,
// 32 lanes x 4 floats, lane 4 g + t holding the hi halves of W[8 nb + g, 8 kb + t, j] and W[8 nb + g, 8 kb + t + 4, j],
// then their lo halves.  They are read through the read-only cache straight into registers, one step ahead of their
// MMAs: every warp of a CTA reads the same ones.  The staged input is split once per chunk, in shared memory.
//
// No atomics and no global mutable state: every output element has one writer and a fixed summation order, so results
// are bit-identical from run to run, and concurrent calls from several host threads are independent.
#ifndef B2D_HOST_EMU               // tests/emu/ runs these kernels' source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif
#include "mma_sync.cuh"
#include "tf32_split.cuh"

namespace {

constexpr int kKC = 16;            // input channels per staged chunk
constexpr int kKS = kKC + 4;       // shared-memory row stride: 8 consecutive rows x 4 columns hit 32 distinct banks
constexpr int kWarps = 4;
constexpr float kLrelu = 0.1f;     // LRELU_SLOPE (models.py:12)

struct HgConvParams {
    const float* x;                // element (b, t, c) at x[b sb + t st + c sc]
    long long sb, st, sc;
    int B, T, Cin;
    const float* w;                // fragment-packed [k][Cin / 8][N / 8][32][4]
    const float* bias;             // [N], or [C_out] for the transposed convolution
    int k, dil, N;
    int lrelu;                     // prologue leaky_relu(., 0.1)
    const float* residual;         // [B, T, N] or NULL
    const float* accum;            // [B, T, N] or NULL
    float div;
    int up;                        // 0: plain; u: polyphase transposed convolution, N = u C_out
    const float* src;              // [B, T_src] (T_src = T u s) or NULL
    const float* wn;               // [C_out, n_k]
    const float* bn;               // [C_out]
    int n_k, n_stride, n_pad;
    float* out;                    // [B, T, N] or [B, T u, C_out]
};

// BM time rows (4 warps of BM / 4 rows, MT m16 tiles each) x BN output columns (NT n8 tiles) per CTA.
// Grid: (ceil(T / BM), N / BN, B).
template <int BM, int BN>
__global__ void __launch_bounds__(kWarps * 32) hg_conv_kernel(HgConvParams p) {
    constexpr int MT = BM / kWarps / 16, NT = BN / 8;
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, tg = lane & 3;
    const int b = blockIdx.z, t0 = blockIdx.x * BM, nb0 = blockIdx.y * (BN / 8);
    const int T = p.T, halo = p.dil * (p.k - 1) / 2, R = BM + 2 * halo;
    const int n_chunks = p.Cin / kKC, KB = p.Cin / 8, NB = p.N / 8;
    const float* xb = p.x + (long long)b * p.sb;
    const bool vec = p.sc == 1;                              // 16-byte copies (the host checked alignment)

    // rows t0 - halo .. t0 + BM + halo - 1, channels of chunk cc -> stage cc & 1; outside [0, T): zeros
    auto load = [&](int cc) {
        float* tile = smem + (cc & 1) * R * kKS;
        const int c0 = cc * kKC;
        if (vec) {
            for (int i = tid; i < R * 4; i += kWarps * 32) {
                const int row = i >> 2, q = i & 3, t = t0 - halo + row;
                const bool in = t >= 0 && t < T;
                const float* s = in ? xb + (long long)t * p.st + c0 + 4 * q : p.x;
                cp_async16(b2d::smem_u32(tile + row * kKS + 4 * q), s, in ? 16u : 0u);
            }
        } else {                                             // strided input (conv_pre on a channel-major mel)
            const bool t_fast = p.st == 1;                   // consecutive threads along the unit stride
            for (int i = tid; i < R * kKC; i += kWarps * 32) {
                const int row = t_fast ? i % R : i / kKC, c = t_fast ? i / R : i % kKC, t = t0 - halo + row;
                tile[row * kKS + c] = (t >= 0 && t < T) ? __ldg(xb + (long long)t * p.st + (long long)(c0 + c) * p.sc)
                                                        : 0.f;
            }
        }
        cp_async_commit();
    };

    float acc[MT][NT][4], part[MT][NT][4];
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int n = 0; n < NT; ++n)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[m][n][e] = 0.f;

    float* lo_tile = smem + 2 * R * kKS;                     // TF32 low halves of the current chunk
    const float4* wf = reinterpret_cast<const float4*>(p.w) + lane;
    load(0);
    for (int cc = 0; cc < n_chunks; ++cc) {
        if (cc + 1 < n_chunks) {
            load(cc + 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        // prologue and TF32 split once per staged element (not once per tap): hi in place, lo beside it
        float* hi_tile = smem + (cc & 1) * R * kKS;
        for (int i = tid; i < R * kKC; i += kWarps * 32) {
            const int o = (i >> 4) * kKS + (i & 15);
            float v = hi_tile[o];
            if (p.lrelu) v = v >= 0.f ? v : v * kLrelu;
            float h, l;
            tf32_split(v, h, l);
            hi_tile[o] = h;
            lo_tile[o] = l;
        }
        __syncthreads();
        const int base = (warp * (BM / kWarps) + g) * kKS + tg;
        const float* th = hi_tile + base;
        const float* tl = lo_tile + base;
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int n = 0; n < NT; ++n)
#pragma unroll
                for (int e = 0; e < 4; ++e) part[m][n][e] = 0.f;
        // B fragments (hi0, hi1, lo0, lo1) of step (j, kk), loaded one step ahead of their MMAs
        auto load_b = [&](float4 (&bq)[NT], int j, int kk) {
            const float4* wk = wf + ((size_t)(j * KB + cc * 2 + kk) * NB + nb0) * 32;
#pragma unroll
            for (int n = 0; n < NT; ++n) bq[n] = __ldg(wk + n * 32);
        };
        auto step = [&](const float4 (&bq)[NT], int j, int kk) {
            uint32_t ah[MT][4], al[MT][4];
#pragma unroll
            for (int m = 0; m < MT; ++m)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    // a0 (row g, col t), a1 (g + 8, t), a2 (g, t + 4), a3 (g + 8, t + 4)
                    const int o = (j * p.dil + m * 16 + (e & 1) * 8) * kKS + kk * 8 + (e >> 1) * 4;
                    ah[m][e] = __float_as_uint(th[o]);
                    al[m][e] = __float_as_uint(tl[o]);
                }
#pragma unroll
            for (int n = 0; n < NT; ++n) {
                const uint32_t bh0 = __float_as_uint(bq[n].x), bh1 = __float_as_uint(bq[n].y);
#pragma unroll
                for (int m = 0; m < MT; ++m) {               // the small terms first
                    mma_tf32(part[m][n], al[m], bh0, bh1);
                    mma_tf32(part[m][n], ah[m], __float_as_uint(bq[n].z), __float_as_uint(bq[n].w));
                    mma_tf32(part[m][n], ah[m], bh0, bh1);
                }
            }
        };
        float4 b0[NT], b1[NT];
        load_b(b0, 0, 0);
#pragma unroll 1
        for (int j = 0; j < p.k; ++j) {
            load_b(b1, j, 1);
            step(b0, j, 0);
            if (j + 1 < p.k) load_b(b0, j + 1, 0);
            step(b1, j, 1);
        }
        // the tensor cores' fp32 accumulation truncates: a chunk's products are summed from zero and added to the total
        // with a rounded add, so the truncation bias does not grow with C_in k
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int n = 0; n < NT; ++n)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[m][n][e] += part[m][n][e];
        __syncthreads();                                     // stage cc & 1 is refilled by the next iteration's load
    }

    // epilogue: acc[m][n][e] is row warp BM / 4 + 16 m + g + 8 (e >> 1), column 8 (nb0 + n) + 2 tg + (e & 1)
    const int Cout = p.up ? p.N / p.up : p.N;
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int t = t0 + warp * (BM / kWarps) + m * 16 + g + 8 * h;
            if (t >= T) continue;
#pragma unroll
            for (int n = 0; n < NT; ++n) {
                const int col = 8 * (nb0 + n) + 2 * tg;
                float v0 = acc[m][n][2 * h], v1 = acc[m][n][2 * h + 1];
                if (!p.up) {
                    const size_t o = ((size_t)b * T + t) * p.N + col;
                    const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + col));
                    v0 += bv.x; v1 += bv.y;
                    if (p.residual) {
                        const float2 r = *reinterpret_cast<const float2*>(p.residual + o);
                        v0 += r.x; v1 += r.y;
                    }
                    if (p.accum) {
                        const float2 a = *reinterpret_cast<const float2*>(p.accum + o);
                        v0 = a.x + v0; v1 = a.y + v1;
                    }
                    *reinterpret_cast<float2*>(p.out + o) = make_float2(v0 / p.div, v1 / p.div);
                } else {
                    const int r = col / Cout, co = col - r * Cout;           // co, co + 1: same phase (C_out even)
                    const long long To = (long long)T * p.up, tout = (long long)t * p.up + r;
                    const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + co));
                    v0 += bv.x; v1 += bv.y;
                    if (p.src) {                                             // noise_convs[i](har_source)
                        const long long Ts = To * p.n_stride, s0 = tout * p.n_stride - p.n_pad;
                        const float* sb = p.src + (long long)b * Ts;
                        const float* w0 = p.wn + (size_t)co * p.n_k;
                        const float* w1 = w0 + p.n_k;
                        float n0 = 0.f, n1 = 0.f;
                        for (int q = 0; q < p.n_k; ++q) {
                            const long long s = s0 + q;
                            if (s < 0 || s >= Ts) continue;
                            const float sv = __ldg(sb + s);
                            n0 = fmaf(__ldg(w0 + q), sv, n0);
                            n1 = fmaf(__ldg(w1 + q), sv, n1);
                        }
                        v0 += n0 + __ldg(p.bn + co);
                        v1 += n1 + __ldg(p.bn + co + 1);
                    }
                    *reinterpret_cast<float2*>(p.out + ((size_t)b * To + tout) * Cout + co) = make_float2(v0, v1);
                }
            }
        }
}

// out[b, 0, t] = tanh(bias[0] + sum_{j < 7, c} w[j][c] leaky_relu(x[b, t + j - 3, c], 0.01)).  One thread per sample; the
// weights [7][C] in shared memory.
__global__ void __launch_bounds__(256) hg_post_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                      const float* __restrict__ bias, int B, int T, int C, float* __restrict__ out) {
    extern __shared__ __align__(16) float sw[];
    for (int i = threadIdx.x; i < 7 * C; i += blockDim.x) sw[i] = w[i];
    __syncthreads();
    // the reference's last leaky_relu takes torch's default slope, 0.01, not LRELU_SLOPE (models.py:260)
    const float slope = 0.01f;
    const long long n = (long long)B * T;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const long long bb = i / T;
        const int t = (int)(i - bb * T);
        float s = 0.f;
        for (int j = 0; j < 7; ++j) {
            const int tt = t + j - 3;
            if (tt < 0 || tt >= T) continue;
            const float4* row = reinterpret_cast<const float4*>(x + (bb * T + tt) * C);
            const float* wj = sw + j * C;
            for (int c4 = 0; c4 < C / 4; ++c4) {
                const float4 v = __ldg(row + c4);
                const float a[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int e = 0; e < 4; ++e) s = fmaf(wj[4 * c4 + e], a[e] >= 0.f ? a[e] : a[e] * slope, s);
            }
        }
        out[i] = tanhf(s + __ldg(bias));
    }
}

#ifndef B2D_HOST_EMU
template <int BM, int BN>
int launch_conv(const HgConvParams& p, cudaStream_t st) {
    const int halo = p.dil * (p.k - 1) / 2;
    const size_t smem = (size_t)3 * (BM + 2 * halo) * kKS * sizeof(float);    // 2 stages + lo
    auto kern = hg_conv_kernel<BM, BN>;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return b2d::fail((int)e, "hifigan_conv: smem attr (%zu B): %s", smem, cudaGetErrorString(e));
    }
    dim3 grid((p.T + BM - 1) / BM, p.N / BN, p.B);
    kern<<<grid, kWarps * 32, smem, st>>>(p);
    return b2d::check_launch("hifigan_conv");
}
#endif  // B2D_HOST_EMU

}  // namespace

#ifndef B2D_HOST_EMU
namespace b2d {

// BN: 32, or 16 when it does not divide N.  BM = 128 rows, or 64 when 128-row tiles would leave the grid under
// two CTAs per SM (short utterances at the wide early stages).
int hifigan_conv_launch(const float* x, int64_t sb, int64_t st_, int64_t sc, int B, int T, int Cin, const float* w,
                        const float* bias, int k, int dil, int N, int lrelu, const float* residual, const float* accum,
                        float div, int up, const float* src, const float* wn, const float* bn, int n_k, int n_stride,
                        int n_pad, float* out, cudaStream_t stream) {
    HgConvParams p{x, sb, st_, sc, B, T, Cin, w, bias, k, dil, N, lrelu, residual, accum, div, up, src, wn, bn,
                   n_k, n_stride, n_pad, out};
    const int BN = N % 32 == 0 ? 32 : 16;
    const long long ctas128 = (long long)((T + 127) / 128) * (N / BN) * B;
    const bool small = ctas128 < 2LL * num_sms();
    switch (BN) {
        case 32: return small ? launch_conv<64, 32>(p, stream) : launch_conv<128, 32>(p, stream);
        default: return small ? launch_conv<64, 16>(p, stream) : launch_conv<128, 16>(p, stream);
    }
}

int hifigan_post_launch(const float* x, const float* w, const float* bias, int B, int T, int C, float* out,
                        cudaStream_t stream) {
    const long long n = (long long)B * T;
    long long grid = (n + 255) / 256;
    const long long cap = (long long)num_sms() * 16;
    hg_post_kernel<<<(unsigned)(grid > cap ? cap : grid), 256, (size_t)7 * C * sizeof(float), stream>>>(x, w, bias, B, T,
                                                                                                         C, out);
    return check_launch("hifigan_post");
}

}  // namespace b2d
#endif  // B2D_HOST_EMU
