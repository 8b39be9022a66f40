// The RMVPE pitch extractor (encoder/rmvpe/: inference.py, model.py, deepunet.py, seq.py, spec.py, utils.py),
// inference, as seven kernels:
//
//   rv_resample  torchaudio's Resample(sr, 16000, lowpass_filter_width = 128): a polyphase sinc-Hann FIR in fp32 FMA.
//                Output sample j new + p is the dot of phase p's taps with the input from j orig - width on (zero
//                outside); the host builds the [new, taps] table.  One thread per output sample.
//   rv_mel       the log-mel of spec.py: stft(n_fft = win = 1024, hop, hann, center, reflect) -> sqrt(re^2 + im^2)
//                (no epsilon) -> 128-row HTK mel basis over each filter's support -> log(clamp(., 1e-5)).  Two real
//                frames per complex 1024-point FFT (fft_smem.cuh), 16 frames per CTA.  Writes the network's input
//                [B, T_pad, 128] and zeros for the frames past n_frames (mel2hidden's constant padding on the log-mel).
//   rv_conv      a k x k convolution (k = 1, 2 or 3) of channel-contiguous [B, T, F, C] activations as an implicit GEMM
//                on the tensor cores (mma.sync m16n8k8, 3xTF32).  A CTA owns a tile of tT frames x tF bins (BM pixels)
//                and BN output columns; per 16-channel chunk it stages the tile plus its halo once with cp.async (zero
//                padding at the T and F edges) and takes every tap from it.  Epilogue: + bias (eval BatchNorm folded on
//                the host), ReLU or sigmoid, + residual, into a channel slice of a wider buffer, so a decoder's concat
//                is never copied.  k = 3: the 3x3 convolutions (padding 1); k = 1: the 1x1 shortcuts and the GEMMs of
//                the head (F = 1); k = 2 with up: ConvTranspose2d(3x3, stride 2, padding 1, output_padding 1) in
//                polyphase form, the four output phases as 4 C_out columns over input offsets {0, 1}^2, interleaved
//                into the [B, 2T, 2F] output.
//   rv_conv_small  direct fp32 convolution for the two ends the tiles do not cover: the first convolution and its 1x1
//                shortcut (C_in = 1, the encoder's input BatchNorm applied to every real input before the zero padding)
//                and `cnn` (C_out = 3), which writes the head's feature layout c F + f.
//   rv_pool      AvgPool2d(2) of an encoder level's output into the next level's input.
//   rv_gru       the BiGRU recurrence: one 8-CTA thread-block cluster per direction (and batch group), each CTA holding
//                32 hidden units' 96 rows of W_hh in registers; every step ends by broadcasting the new h through
//                distributed shared memory and one cluster barrier.  fp32 FMA.
//   rv_decode    to_local_average_f0: argmax (first index on ties), the +-4-bin weighted mean of the cents, 10 2^(c/1200),
//                zero below the threshold.  One warp per frame.
//
// No atomics and no global mutable state: every output element has one writer and a fixed summation order, so results
// are bit-identical from run to run.
#ifndef B2D_HOST_EMU               // tests/emu/ runs these kernels' source on the CPU (host_emu.h provides the shims)
#include <cooperative_groups.h>

#include "b2d_common.cuh"
#endif
#include "fft_smem.cuh"
#include "mma_sync.cuh"
#include "tf32_split.cuh"

namespace {

namespace cg = cooperative_groups;

// ---------------------------------------------------------------------------------------------------------------------
// rv_conv
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kKC = 16;            // input channels per staged chunk
constexpr int kKS = kKC + 4;       // shared-memory pixel stride: 8 consecutive pixels x 4 columns hit 32 distinct banks
constexpr int kWarps = 4;

struct RvConvParams {
    const float* x;                // element (b, t, f, c) at x[((b T + t) F + f) ldx + c]
    int ldx, B, T, F, Cin;
    const float* w;                // fragment-packed [k k][Cin / 8][N / 8][32][4]
    const float* bias;             // [N], or [N / 4] with up
    int k, N, n_valid, act, up;    // act: 0 none, 1 relu, 2 sigmoid
    const float* res;              // + res[pixel ldr + col] after the activation, or NULL
    int ldr;
    float* out;                    // out[pixel ldo + col]; with up, pixel of the [B, 2T, 2F] grid
    int ldo;
    int tT, tF;                    // pixel tile: tT frames x tF bins, tT tF = BM
};

// BM pixels (4 warps of BM / 4 rows, MT m16 tiles each) x BN output columns (NT n8 tiles) per CTA.
// Grid: ((ceil(T / tT)) (F / tF), N / BN, B).
template <int BM, int BN>
__global__ void __launch_bounds__(kWarps * 32) rv_conv_kernel(RvConvParams p) {
    constexpr int MT = BM / kWarps / 16, NT = BN / 8;
    extern __shared__ __align__(16) float smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, tg = lane & 3;
    const int nft = p.F / p.tF;
    const int b = blockIdx.z, t0 = (blockIdx.x / nft) * p.tT, f0 = (blockIdx.x % nft) * p.tF, nb0 = blockIdx.y * (BN / 8);
    const int hl = p.k == 3, hr = p.k >= 2;                  // halo before / after the tile
    const int W = p.tF + hl + hr, R = (p.tT + hl + hr) * W;
    const int n_chunks = p.Cin / kKC, KB = p.Cin / 8, NB = p.N / 8, taps = p.k * p.k;
    const float* xb = p.x + (size_t)b * p.T * p.F * p.ldx;

    // tile pixels (t0 - hl + i, f0 - hl + j), channels of chunk cc -> stage cc & 1; outside the image: zeros
    auto load = [&](int cc) {
        float* tile = smem + (cc & 1) * R * kKS;
        const int c0 = cc * kKC;
        for (int i = tid; i < R * 4; i += kWarps * 32) {
            const int px = i >> 2, q = i & 3, it = px / W, jf = px - it * W;
            const int t = t0 - hl + it, f = f0 - hl + jf;
            const bool in = t >= 0 && t < p.T && f >= 0 && f < p.F;
            const float* s = in ? xb + ((size_t)t * p.F + f) * p.ldx + c0 + 4 * q : p.x;
            cp_async16(b2d::smem_u32(tile + px * kKS + 4 * q), s, in ? 16u : 0u);
        }
        cp_async_commit();
    };

    // tile offset of this thread's fragment rows g (h = 0) and g + 8 (h = 1) of each m16 tile
    int rbase[MT][2];
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int pr = warp * (BM / kWarps) + m * 16 + g + 8 * h;
            rbase[m][h] = ((pr / p.tF) * W + pr % p.tF) * kKS + tg;
        }

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
        float* hi_tile = smem + (cc & 1) * R * kKS;
        for (int i = tid; i < R * kKC; i += kWarps * 32) {
            const int o = (i >> 4) * kKS + (i & 15);
            float h, l;
            tf32_split(hi_tile[o], h, l);
            hi_tile[o] = h;
            lo_tile[o] = l;
        }
        __syncthreads();
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int n = 0; n < NT; ++n)
#pragma unroll
                for (int e = 0; e < 4; ++e) part[m][n][e] = 0.f;
        auto load_b = [&](float4 (&bq)[NT], int j, int kk) {
            const float4* wk = wf + ((size_t)(j * KB + cc * 2 + kk) * NB + nb0) * 32;
#pragma unroll
            for (int n = 0; n < NT; ++n) bq[n] = __ldg(wk + n * 32);
        };
        auto step = [&](const float4 (&bq)[NT], int toff, int kk) {
            uint32_t ah[MT][4], al[MT][4];
#pragma unroll
            for (int m = 0; m < MT; ++m)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    // a0 (row g, col t), a1 (g + 8, t), a2 (g, t + 4), a3 (g + 8, t + 4)
                    const int o = rbase[m][e & 1] + toff + kk * 8 + (e >> 1) * 4;
                    ah[m][e] = __float_as_uint(hi_tile[o]);
                    al[m][e] = __float_as_uint(lo_tile[o]);
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
        for (int j = 0; j < taps; ++j) {
            const int dt = j / p.k, toff = (dt * W + j - dt * p.k) * kKS;
            load_b(b1, j, 1);
            step(b0, toff, 0);
            if (j + 1 < taps) load_b(b0, j + 1, 0);
            step(b1, toff, 1);
        }
        // the tensor cores' fp32 accumulation truncates: each chunk is summed from zero and added with a rounded add
#pragma unroll
        for (int m = 0; m < MT; ++m)
#pragma unroll
            for (int n = 0; n < NT; ++n)
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[m][n][e] += part[m][n][e];
        __syncthreads();                                     // stage cc & 1 is refilled by the next iteration's load
    }

    // epilogue: acc[m][n][e] is tile pixel warp BM / 4 + 16 m + g + 8 (e >> 1), column 8 (nb0 + n) + 2 tg + (e & 1)
    const int Cout = p.up ? p.N / 4 : p.N;
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int pr = warp * (BM / kWarps) + m * 16 + g + 8 * h;
            const int t = t0 + pr / p.tF, f = f0 + pr % p.tF;
            if (t >= p.T) continue;
            const size_t pix = ((size_t)b * p.T + t) * p.F + f;
#pragma unroll
            for (int n = 0; n < NT; ++n) {
                const int col = 8 * (nb0 + n) + 2 * tg;
                if (col >= p.n_valid) continue;              // n_valid is even: col + 1 is valid too
                float v0 = acc[m][n][2 * h], v1 = acc[m][n][2 * h + 1];
                size_t o;
                int bc = col;
                if (p.up) {                                  // phase r = 2 a + c -> output pixel (2t + a, 2f + c)
                    const int r = col / Cout, a = r >> 1, c = r & 1;
                    bc = col - r * Cout;
                    o = (((size_t)b * 2 * p.T + 2 * t + a) * (2 * p.F) + 2 * f + c) * p.ldo + bc;
                } else {
                    o = pix * p.ldo + col;
                }
                const float2 bv = __ldg(reinterpret_cast<const float2*>(p.bias + bc));
                v0 += bv.x; v1 += bv.y;
                if (p.act == 1) {
                    v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f);
                } else if (p.act == 2) {
                    v0 = 1.f / (1.f + expf(-v0)); v1 = 1.f / (1.f + expf(-v1));
                }
                if (p.res) {
                    const float2 r = *reinterpret_cast<const float2*>(p.res + pix * p.ldr + col);
                    v0 += r.x; v1 += r.y;
                }
                *reinterpret_cast<float2*>(p.out + o) = make_float2(v0, v1);
            }
        }
}

#ifndef B2D_HOST_EMU
template <int BM, int BN>
int launch_conv(RvConvParams p, cudaStream_t st) {
    p.tF = p.F < BM / 4 ? p.F : BM / 4;
    p.tT = BM / p.tF;
    const int hal = (p.k == 3) + (p.k >= 2);
    const size_t smem = (size_t)3 * (p.tT + hal) * (p.tF + hal) * kKS * sizeof(float);    // 2 stages + lo
    // the largest tile of this instantiation is tF = 1 with a halo on both sides: (BM + 2) x 3 pixels.  The opt-in
    // limit is always set to that one value, so concurrent launches from several host threads never lower it under
    // one another's launch.
    constexpr size_t kMaxSmem = (size_t)3 * (BM + 2) * 3 * kKS * sizeof(float);
    auto kern = rv_conv_kernel<BM, BN>;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxSmem);
        if (e != cudaSuccess)
            return b2d::fail((int)e, "rmvpe_conv: smem attr (%zu B): %s", kMaxSmem, cudaGetErrorString(e));
    }
    dim3 grid((unsigned)(((p.T + p.tT - 1) / p.tT) * (p.F / p.tF)), p.N / BN, p.B);
    kern<<<grid, kWarps * 32, smem, st>>>(p);
    return b2d::check_launch("rmvpe_conv");
}
#endif  // B2D_HOST_EMU

// ---------------------------------------------------------------------------------------------------------------------
// rv_conv_small: one thread per output pixel, every output channel
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kSmallMaxCout = 16;

struct RvSmallParams {
    const float* x;                // element (b, t, f, c) at x[b sb + t st + f sf + c sc]
    long long sb, st, sf, sc;
    int B, T, F, Cin;
    const float* in_scale;         // x c -> x in_scale[c] + in_shift[c] on real pixels (eval BatchNorm), or NULL
    const float* in_shift;
    const float* w;                // [Cout][Cin][k][k]
    const float* bias;             // [Cout] or NULL
    int k, Cout, act, head;        // head: out[((b T + t) Cout + co) F + f]; else out[pixel ldo + co]
    float* out;
    int ldo;
};

__global__ void __launch_bounds__(128) rv_conv_small_kernel(RvSmallParams p) {
    extern __shared__ __align__(16) float sw[];
    const int nw = p.Cout * p.Cin * p.k * p.k;
    for (int i = threadIdx.x; i < nw; i += blockDim.x) sw[i] = p.w[i];
    __syncthreads();
    const long long n = (long long)p.B * p.T * p.F;
    const int org = p.k == 3 ? -1 : 0, kk = p.k * p.k;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int f = (int)(i % p.F);
        const long long bt = i / p.F;
        const int t = (int)(bt % p.T), b = (int)(bt / p.T);
        float acc[kSmallMaxCout];
#pragma unroll
        for (int co = 0; co < kSmallMaxCout; ++co) acc[co] = 0.f;
        for (int dt = 0; dt < p.k; ++dt) {
            const int tt = t + org + dt;
            if (tt < 0 || tt >= p.T) continue;
            for (int df = 0; df < p.k; ++df) {
                const int ff = f + org + df;
                if (ff < 0 || ff >= p.F) continue;
                const float* xp = p.x + b * p.sb + tt * p.st + ff * p.sf;
                for (int ci = 0; ci < p.Cin; ++ci) {
                    float v = __ldg(xp + ci * p.sc);
                    if (p.in_scale) v = fmaf(v, __ldg(p.in_scale + ci), __ldg(p.in_shift + ci));
                    const float* wc = sw + ci * kk + dt * p.k + df;
#pragma unroll
                    for (int co = 0; co < kSmallMaxCout; ++co)
                        if (co < p.Cout) acc[co] = fmaf(wc[co * p.Cin * kk], v, acc[co]);
                }
            }
        }
#pragma unroll
        for (int co = 0; co < kSmallMaxCout; ++co) {
            if (co >= p.Cout) break;
            float v = acc[co] + (p.bias ? __ldg(p.bias + co) : 0.f);
            if (p.act) v = fmaxf(v, 0.f);
            if (p.head) p.out[(bt * p.Cout + co) * p.F + f] = v;
            else p.out[i * p.ldo + co] = v;
        }
    }
}

// out [B, T/2, F/2, C] = AvgPool2d(2) of x (element (b, t, f, c) at x[((b T + t) F + f) ldx + c]); one thread per output
__global__ void __launch_bounds__(256) rv_pool_kernel(const float* __restrict__ x, int ldx, int B, int T, int F, int C,
                                                      float* __restrict__ out) {
    const int To = T / 2, Fo = F / 2;
    const long long n = (long long)B * To * Fo * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        long long r = i / C;
        const int f = (int)(r % Fo);
        r /= Fo;
        const int t = (int)(r % To), b = (int)(r / To);
        const float* p0 = x + (((size_t)b * T + 2 * t) * F + 2 * f) * ldx + c;
        const float* p1 = p0 + (size_t)F * ldx;
        out[i] = (__ldg(p0) + __ldg(p0 + ldx) + __ldg(p1) + __ldg(p1 + ldx)) * 0.25f;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// rv_gru: nn.GRU(384, 256, batch_first, bidirectional) recurrence after the input projection
//   r = sigmoid(xr + W_hr h + b_hr), z = sigmoid(xz + W_hz h + b_hz), n = tanh(xn + r (W_hn h + b_hn)),
//   h' = n + z (h - n)  (torch's gate order r, z, n; xg = W_ih x + b_ih from rv_conv)
// Grid (16, ceil(B / kGruB)): CTAs 0-7 the forward direction, 8-15 the backward one, one cluster of 8 each.  CTA rank q
// owns hidden units [32 q, 32 q + 32); warp w of it units 32 q + 4 w + j (j < 4) and their rows r, z, n: 12 rows of
// W_hh, lane l holding columns l + 32 c (c < 8) in registers.  The partial dots are summed across the warp by an xor
// butterfly, so every lane holds the same 12 sums.  h lives in every CTA's shared memory, double-buffered by step parity:
// a step reads buffer s & 1 and writes the new h slice into buffer (s + 1) & 1 of all 8 CTAs, and the one cluster barrier
// at its end orders both.
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kGruH = 256, kGruCta = 8, kGruB = 4, kGruThreads = 256;

__global__ void __cluster_dims__(kGruCta, 1, 1) __launch_bounds__(kGruThreads, 1)
    rv_gru_kernel(const float* __restrict__ xg, const float* __restrict__ whh, const float* __restrict__ bhh, int B,
                  int T, float* __restrict__ out) {
    cg::cluster_group cluster = cg::this_cluster();
    B2D_SHARED(float, hbuf, [2][kGruB][kGruH]);
    B2D_SHARED(float, red, [kGruThreads / 32][kGruB][12]);
    const int rank = (int)cluster.block_rank(), dir = blockIdx.x / kGruCta;
    const int b0 = blockIdx.y * kGruB, nb = min(kGruB, B - b0);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int u0 = rank * (kGruH / kGruCta) + warp * 4;

    float wr[12][8];
    const float* wd = whh + (size_t)dir * 3 * kGruH * kGruH;
#pragma unroll
    for (int i = 0; i < 12; ++i)
#pragma unroll
        for (int c = 0; c < 8; ++c) wr[i][c] = __ldg(wd + (size_t)((i >> 2) * kGruH + u0 + (i & 3)) * kGruH + lane + 32 * c);
    // gate step: lane 4 bb + jj owns (utterance b0 + bb, unit u0 + jj)
    const int bb = lane >> 2, jj = lane & 3, unit = u0 + jj;
    const bool owner = bb < nb;
    float bh[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) bh[q] = __ldg(bhh + dir * 3 * kGruH + q * kGruH + unit);
    for (int i = threadIdx.x; i < 2 * kGruB * kGruH; i += kGruThreads) (&hbuf[0][0][0])[i] = 0.f;
    cluster.sync();                                          // every CTA of the cluster runs and its h is zero

    const int G = 2 * 3 * kGruH;                             // xg row: [direction][gate][unit]
    for (int s = 0; s < T; ++s) {
        const int t = dir ? T - 1 - s : s, cur = s & 1;
        float xr = 0.f, xz = 0.f, xn = 0.f;
        if (owner) {
            const float* xrow = xg + ((size_t)(b0 + bb) * T + t) * G + dir * 3 * kGruH + unit;
            xr = __ldg(xrow); xz = __ldg(xrow + kGruH); xn = __ldg(xrow + 2 * kGruH);
        }
        for (int b = 0; b < nb; ++b) {
            float hv[8];
#pragma unroll
            for (int c = 0; c < 8; ++c) hv[c] = hbuf[cur][b][lane + 32 * c];
#pragma unroll
            for (int i = 0; i < 12; ++i) {
                float v = 0.f;
#pragma unroll
                for (int c = 0; c < 8; ++c) v = fmaf(wr[i][c], hv[c], v);
#pragma unroll
                for (int off = 16; off; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
                if (lane == 0) red[warp][b][i] = v;
            }
        }
        __syncwarp();
        if (owner) {
            const float hr = red[warp][bb][jj] + bh[0], hz = red[warp][bb][4 + jj] + bh[1];
            const float hn = red[warp][bb][8 + jj] + bh[2];
            const float r = 1.f / (1.f + expf(-(xr + hr))), z = 1.f / (1.f + expf(-(xz + hz)));
            const float n = tanhf(xn + r * hn);
            const float hp = hbuf[cur][bb][unit];
            const float h = n + z * (hp - n);
            out[((size_t)(b0 + bb) * T + t) * (2 * kGruH) + dir * kGruH + unit] = h;
#pragma unroll
            for (int q = 0; q < kGruCta; ++q) *cluster.map_shared_rank(&hbuf[cur ^ 1][bb][unit], q) = h;
        }
        cluster.sync();
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// rv_resample
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rv_resample_kernel(const float* __restrict__ x, int B, int N,
                                                          const float* __restrict__ table, int nw, int orig, int taps,
                                                          int width, int n_out, float* __restrict__ out) {
    const long long n = (long long)B * n_out;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i / n_out), o = (int)(i - (long long)b * n_out);
        const int j = o / nw, ph = o - j * nw;
        const long long s0 = (long long)j * orig - width;    // input sample of tap 0
        const int k0 = s0 < 0 ? (int)-s0 : 0;
        const long long kend = (long long)N - s0;
        const int k1 = kend < taps ? (int)kend : taps;
        const float* w = table + (size_t)ph * taps;
        const float* xs = x + (size_t)b * N + s0;
        float acc = 0.f;
        for (int k = k0; k < k1; ++k) acc = fmaf(__ldg(w + k), __ldg(xs + k), acc);
        out[i] = acc;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// rv_mel
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kMelN = 1024, kMelBins = kMelN / 2 + 1, kMelRows = 128, kMelFrames = 16;
constexpr int kMelPad = b2d_fft_smem::Plan<kMelN>::kPad, kMelTw2 = b2d_fft_smem::Plan<kMelN>::kTw2;
constexpr int kMelTw3 = b2d_fft_smem::Plan<kMelN>::kTw3, kMagStride = kMelBins + 3;
constexpr size_t kMelSmem = (size_t)(kMelPad + kMelTw2 + kMelTw3) * sizeof(float2) + (size_t)2 * kMagStride * sizeof(float);
static_assert(b2d_fft_smem::kThreads == kMelRows, "one thread per mel row");

struct RvMelParams {
    const float* y;                // [B, N]
    const float* window;           // [1024] hann (periodic)
    const float* basis;            // [128, 513]
    const int* lohi;               // [128, 2] support of each filter
    float* out;                    // [B, t_pad, 128]
    int N, hop, n_frames, t_pad;
};

__device__ __forceinline__ float reflect_at(const float* __restrict__ y, int N, int s) {
    if (s < 0) s = -s;                                       // torch 'reflect' (pad < N is checked on the host)
    else if (s >= N) s = 2 * (N - 1) - s;
    return __ldg(y + s);
}

__global__ void __launch_bounds__(b2d_fft_smem::kThreads) rv_mel_kernel(RvMelParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* Fz = reinterpret_cast<float2*>(smem_raw);
    float2* tw2 = Fz + kMelPad;
    float2* tw3 = tw2 + kMelTw2;
    float* mag = reinterpret_cast<float*>(tw3 + kMelTw3);    // [2][kMagStride]
    const int tid = threadIdx.x, b = blockIdx.y;
    const int fr0 = blockIdx.x * kMelFrames;
    const int fr1 = min(fr0 + kMelFrames, p.t_pad), fr_real = min(fr1, p.n_frames);
    const float* y = p.y + (size_t)b * p.N;
    float* ob = p.out + (size_t)b * p.t_pad * kMelRows;

    b2d_fft_smem::init_twiddles<kMelN>(tw2, tw3, tid);
    const int lo = __ldg(p.lohi + 2 * tid), hi = __ldg(p.lohi + 2 * tid + 1);
    const float* brow = p.basis + (size_t)tid * kMelBins;
    for (int fa = fr0; fa < fr_real; fa += 2) {
        const bool has_b = fa + 1 < fr_real;
        const int s0 = fa * p.hop - kMelN / 2;
        for (int u = 0; u < kMelN / b2d_fft_smem::kThreads; ++u) {
            const int n = tid + u * b2d_fft_smem::kThreads;
            const float w = __ldg(p.window + n);
            const float va = reflect_at(y, p.N, s0 + n);
            const float vb = has_b ? reflect_at(y, p.N, s0 + p.hop + n) : 0.f;
            Fz[b2d_fft_smem::padi(n)] = make_float2(w * va, w * vb);
        }
        __syncthreads();
        b2d_fft_smem::fft_forward<kMelN, 1, true>(Fz, tw2, tw3, tid);
        for (int k = tid; k < kMelBins; k += b2d_fft_smem::kThreads) {
            // A = (Z[k] + conj Z[N-k]) / 2, B = (Z[k] - conj Z[N-k]) / 2j
            const float2 zk = Fz[b2d_fft_smem::padi(k)], zm = Fz[b2d_fft_smem::padi((kMelN - k) & (kMelN - 1))];
            const float ar = 0.5f * (zk.x + zm.x), ai = 0.5f * (zk.y - zm.y);
            const float br = 0.5f * (zk.y + zm.y), bi = 0.5f * (zm.x - zk.x);
            mag[k] = sqrtf(ar * ar + ai * ai);
            mag[kMagStride + k] = sqrtf(br * br + bi * bi);
        }
        __syncthreads();
        float sa = 0.f, sb = 0.f;
        for (int k = lo; k < hi; ++k) {
            const float wgt = __ldg(brow + k);
            sa = fmaf(wgt, mag[k], sa);
            sb = fmaf(wgt, mag[kMagStride + k], sb);
        }
        ob[(size_t)fa * kMelRows + tid] = logf(fmaxf(sa, 1e-5f));
        if (has_b) ob[(size_t)(fa + 1) * kMelRows + tid] = logf(fmaxf(sb, 1e-5f));
        // the next pair's loads write Fz only; mag is rewritten after two more barriers
    }
    for (int fa = max(fr0, fr_real); fa < fr1; ++fa) ob[(size_t)fa * kMelRows + tid] = 0.f;
}

// ---------------------------------------------------------------------------------------------------------------------
// rv_decode: sal [B, t_pad, 360] -> f0 [B, n_frames]; one warp per frame
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kClasses = 360;
constexpr float kCents0 = 1997.3794084376191f;

__global__ void __launch_bounds__(256) rv_decode_kernel(const float* __restrict__ sal, int B, int t_pad, int n_frames,
                                                        float thred, float* __restrict__ f0) {
    const int lane = threadIdx.x & 31;
    const long long n = (long long)B * n_frames;
    const long long warps = (long long)gridDim.x * (blockDim.x / 32);
    for (long long i = (long long)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); i < n; i += warps) {
        const int b = (int)(i / n_frames), t = (int)(i - (long long)b * n_frames);
        const float* s = sal + ((size_t)b * t_pad + t) * kClasses;
        float best = -INFINITY;
        int bi = 0;
        for (int c = lane; c < kClasses; c += 32) {
            const float v = __ldg(s + c);
            if (v > best) { best = v; bi = c; }
        }
        for (int off = 16; off; off >>= 1) {                 // the first index among equal maxima, as torch.argmax
            const float ob = __shfl_xor_sync(0xffffffffu, best, off);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
            if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
        }
        if (lane == 0) {
            const int c0 = max(0, bi - 4), c1 = min(kClasses, bi + 5);
            float ws = 0.f, ps = 0.f;
            for (int c = c0; c < c1; ++c) {
                const float v = __ldg(s + c);
                ws += v;
                ps = fmaf(v, (float)(20 * c) + kCents0, ps);
            }
            const float cents = ps / (ws + (ws == 0.f ? 1.f : 0.f));
            f0[i] = best < thred ? 0.f : 10.f * exp2f(cents / 1200.f);
        }
    }
}

#ifndef B2D_HOST_EMU
unsigned grid_for(long long n, int threads) {
    const long long g = (n + threads - 1) / threads, cap = (long long)b2d::num_sms() * 16;
    return (unsigned)(g < 1 ? 1 : (g > cap ? cap : g));
}
#endif  // B2D_HOST_EMU

}  // namespace

#ifndef B2D_HOST_EMU
namespace b2d {

// BN: 32, or 16 when it does not divide N.  BM = 128 pixels, or 64 when 128-pixel tiles would leave the grid under two
// CTAs per SM (the deep levels at small batches).
int rmvpe_conv_launch(const float* x, int ldx, int B, int T, int F, int Cin, const float* w, const float* bias, int k,
                      int N, int n_valid, int act, int up, const float* res, int ldr, float* out, int ldo,
                      cudaStream_t stream) {
    RvConvParams p{x, ldx, B, T, F, Cin, w, bias, k, N, n_valid, act, up, res, ldr, out, ldo, 0, 0};
    const int BN = N % 32 == 0 ? 32 : 16;
    const long long ctas128 = ((long long)T * F + 127) / 128 * (N / BN) * B;
    const bool small = ctas128 < 2LL * num_sms();
    switch (BN) {
        case 32: return small ? launch_conv<64, 32>(p, stream) : launch_conv<128, 32>(p, stream);
        default: return small ? launch_conv<64, 16>(p, stream) : launch_conv<128, 16>(p, stream);
    }
}

int rmvpe_conv_small_launch(const float* x, int64_t sb, int64_t st, int64_t sf, int64_t sc, int B, int T, int F, int Cin,
                            const float* in_scale, const float* in_shift, const float* w, const float* bias, int k,
                            int Cout, int act, int head, float* out, int ldo, cudaStream_t stream) {
    RvSmallParams p{x, sb, st, sf, sc, B, T, F, Cin, in_scale, in_shift, w, bias, k, Cout, act, head, out, ldo};
    const size_t smem = (size_t)Cout * Cin * k * k * sizeof(float);
    rv_conv_small_kernel<<<grid_for((long long)B * T * F, 128), 128, smem, stream>>>(p);
    return check_launch("rmvpe_conv_small");
}

int rmvpe_pool_launch(const float* x, int ldx, int B, int T, int F, int C, float* out, cudaStream_t stream) {
    rv_pool_kernel<<<grid_for((long long)B * (T / 2) * (F / 2) * C, 256), 256, 0, stream>>>(x, ldx, B, T, F, C, out);
    return check_launch("rmvpe_pool");
}

int rmvpe_gru_launch(const float* xg, const float* whh, const float* bhh, int B, int T, float* out, cudaStream_t stream) {
    dim3 grid(2 * kGruCta, (B + kGruB - 1) / kGruB);
    rv_gru_kernel<<<grid, kGruThreads, 0, stream>>>(xg, whh, bhh, B, T, out);
    return check_launch("rmvpe_gru");
}

int rmvpe_resample_launch(const float* x, int B, int N, const float* table, int new_freq, int orig_freq, int taps,
                          int width, int n_out, float* out, cudaStream_t stream) {
    rv_resample_kernel<<<grid_for((long long)B * n_out, 256), 256, 0, stream>>>(x, B, N, table, new_freq, orig_freq,
                                                                               taps, width, n_out, out);
    return check_launch("rmvpe_resample");
}

int rmvpe_mel_launch(const float* y, int B, int N, const float* window, const float* basis, const int* lohi, int hop,
                     int n_frames, int t_pad, float* out, cudaStream_t stream) {
    RvMelParams p{y, window, basis, lohi, out, N, hop, n_frames, t_pad};
    static_assert(kMelSmem <= 48 * 1024, "no opt-in shared memory needed");
    dim3 grid((t_pad + kMelFrames - 1) / kMelFrames, B);
    rv_mel_kernel<<<grid, b2d_fft_smem::kThreads, kMelSmem, stream>>>(p);
    return check_launch("rmvpe_mel");
}

int rmvpe_decode_launch(const float* sal, int B, int t_pad, int n_frames, float thred, float* f0, cudaStream_t stream) {
    rv_decode_kernel<<<grid_for((long long)B * n_frames * 32, 256), 256, 0, stream>>>(sal, B, t_pad, n_frames, thred, f0);
    return check_launch("rmvpe_decode");
}

}  // namespace b2d
#endif  // B2D_HOST_EMU
