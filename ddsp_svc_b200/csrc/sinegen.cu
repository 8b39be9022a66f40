// K6: NSF-HiFiGAN SineGen f0 excitation  (reference nsf_hifigan/models.py:134-165).
//
//   out[b, t, h] = sine_amp * sin(2 pi ((h+1) rad[t] + rho_h)) * uv[t] + noise_amp[t] * eps[b,t,h]
//   rad[k*upp + j] = (f0[k]/sr) (j+1) + acc[k-1],   acc = per-frame wrapped phase advance
//   uv = 1[f0[k] > thr],  noise_amp = uv*noise_std + (1-uv)*sine_amp/3,  eps ~ N(0,1)
//
// The reference evaluates everything in fp32 (piecewise-constant f0, fmod-wrapped frame advance
// accumulated by a cumsum that -- on CPU, the oracle -- accumulates in fp64 and emits fp32); the
// operation order below mirrors it so results agree to the last few ulps of the sin argument.
//
// Two launches: (1) a per-utterance frame scan (n_frames values); (2) the streaming kernel.
// (2) is write-bound (dim*4 = 36 B per audio sample): a CTA owns 128 consecutive samples x dim
// harmonics, each thread computes the `dim` values of one sample into shared memory, and the tile
// is written back as coalesced 128-bit stores.  Noise is either read (parity mode, same tiling)
// or generated in-kernel: Philox4x32-10 + Box-Muller, keyed by (seed, utterance, flat index).
#include "b2d_common.cuh"

namespace {

constexpr int kScanThreads = 256;
constexpr int kTile = 128;   // samples per CTA
constexpr int kMaxDim = 16;

// acc_prev[b,k] = fp32( fmod( fp32( sum_{i<k} adv_i ), 1 ) ),  adv_i = fmod(s_i*upp + 0.5, 1) - 0.5
__global__ void __launch_bounds__(kScanThreads)
sinegen_scan_kernel(const float* __restrict__ f0, int nF, int upp, float sr, float* __restrict__ acc_prev) {
    const int b = blockIdx.x;
    const float* f = f0 + (size_t)b * nF;
    const int per = (nF + kScanThreads - 1) / kScanThreads;
    const int k0 = min(nF, (int)threadIdx.x * per), k1 = min(nF, k0 + per);
    const float fupp = (float)upp;
    auto adv = [&](int k) {
        const float s = __fdiv_rn(f[k], sr);
        const float last = __fmul_rn(s, fupp);                       // rad[k, upp-1]
        return __fsub_rn(fmodf(__fadd_rn(last, 0.5f), 1.0f), 0.5f);  // (:139)
    };
    double local = 0.0;
    for (int k = k0; k < k1; ++k) local += (double)adv(k);
    __shared__ double warp_tot[kScanThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double incl = local;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        double up = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += up;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    double run = incl - local;
    for (int w = 0; w < warp; ++w) run += warp_tot[w];
    for (int k = k0; k < k1; ++k) {
        // exclusive: what the reference adds to frame k is fmod(cumsum[k-1], 1)   (:140-141)
        acc_prev[(size_t)b * nF + k] = (k == 0) ? 0.0f : fmodf((float)run, 1.0f);
        run += (double)adv(k);
    }
}

struct SgParams {
    const float* f0;
    const float* acc_prev;
    const float* rand_ini;  // [dim]
    const float* noise_in;  // [B, T, dim] or nullptr
    float* out;             // [B, T, dim]
    int nF, upp, dim;
    int upp_shift;          // log2(upp) if upp is a power of two, else -1
    float sr, sine_amp;
    float namp_voiced, namp_unvoiced;   // uv*noise_std + (1-uv)*sine_amp/3 for uv = 1 / 0 (fp32, reference op order)
    float thr;
    unsigned long long seed;
    long long utt_off;
    // fused SourceModuleHnNSF tail (nsf_hifigan/models.py:201-204): merged[b,t] = tanh(lin_b + sum_h lin_w[h] out[b,t,h]);
    // when `merged` is set the [B,T,dim] tensor is never written
    const float* lin_w;     // [dim] or nullptr
    float lin_b;
    float* merged;          // [B, T] or nullptr
};

// sin(arg) for |arg| up to a few thousand rad: two-term Cody-Waite reduction, then the SFU.
__device__ __forceinline__ float sin_reduced(float arg) {
    const float k = rintf(arg * 0.15915494309189535f);
    float r = fmaf(k, -6.2831854820251465f, arg);   // 2pi hi (fp32)
    r = fmaf(k, 1.7484555e-7f, r);                  // -(2pi - hi)
    return __sinf(r);
}

// DIM > 0: compile-time number of harmonics (fully unrolled, no predication); DIM == 0: runtime p.dim <= 16
template <int DIM>
__global__ void __launch_bounds__(kTile) sinegen_kernel(SgParams p) {
    extern __shared__ __align__(16) float tile[];  // [kTile * dim]
    constexpr int MAXD = DIM > 0 ? DIM : kMaxDim;
    const int dim = DIM > 0 ? DIM : p.dim;
    const int b = blockIdx.y;
    const int T = p.nF * p.upp;
    const int t0 = blockIdx.x * kTile;
    const int nt = min(kTile, T - t0);
    const int tid = threadIdx.x;
    const size_t base = ((size_t)b * T + t0) * dim;
    const int nflat = nt * dim;

    if (p.noise_in) {  // stage the noise tile (coalesced)
        const float* src = p.noise_in + base;
        if ((base & 3) == 0 && (nflat & 3) == 0) {
            for (int i = tid; i < (nflat >> 2); i += kTile)
                reinterpret_cast<float4*>(tile)[i] = __ldg(reinterpret_cast<const float4*>(src) + i);
        } else {
            for (int i = tid; i < nflat; i += kTile) tile[i] = src[i];
        }
        __syncthreads();
    }

    if (tid < nt) {
        const int t = t0 + tid;
        int k, j;
        if (p.upp_shift >= 0) { k = t >> p.upp_shift; j = t & (p.upp - 1); }
        else { k = t / p.upp; j = t - k * p.upp; }
        const float f = p.f0[(size_t)b * p.nF + k];
        const float s = __fdiv_rn(f, p.sr);                                             // f0 / sr
        const float rad = __fadd_rn(__fmul_rn(s, (float)(j + 1)), p.acc_prev[(size_t)b * p.nF + k]);  // (:138,141)
        const bool voiced = f > p.thr;
        const float namp = voiced ? p.namp_voiced : p.namp_unvoiced;                    // (:162)
        const float samp_uv = voiced ? p.sine_amp : 0.0f;   // (sin*sine_amp)*uv == sin*(sine_amp*uv) for uv in {0,1}
        float* row = tile + tid * dim;
        float eps[MAXD + 3];
        if (p.noise_in) {
#pragma unroll
            for (int h = 0; h < MAXD; ++h) if (h < dim) eps[h] = row[h];
        } else {
            // 4 normals per Philox call; counter = (sample index, call index), key = seed,
            // stream = utterance.  ceil(dim/4) calls per sample (3 for dim = 9; 3 normals unused).
            const unsigned long long utt = (unsigned long long)(p.utt_off + b);
#pragma unroll
            for (int c = 0; c < (MAXD + 3) / 4; ++c) {
                if (4 * c < dim) {
                    uint4 r = b2d::philox4x32_10(make_uint4((uint32_t)t, 0x51e6e000u + c, (uint32_t)utt, (uint32_t)(utt >> 32)),
                                                 make_uint2((uint32_t)p.seed, (uint32_t)(p.seed >> 32)));
                    // Box-Muller: u1,u3 in (0,1], u2,u4 in [0,1);  sqrt(a) = a * rsqrt(a), a > 0
                    const float u1 = ((float)(r.x >> 8) + 1.0f) * (1.0f / 16777216.0f);
                    const float u2 = (float)(r.y >> 8) * (1.0f / 16777216.0f);
                    const float u3 = ((float)(r.z >> 8) + 1.0f) * (1.0f / 16777216.0f);
                    const float u4 = (float)(r.w >> 8) * (1.0f / 16777216.0f);
                    const float a1 = fmaxf(-2.0f * __logf(u1), 1e-30f), a3 = fmaxf(-2.0f * __logf(u3), 1e-30f);
                    const float m1 = a1 * rsqrtf(a1), m2 = a3 * rsqrtf(a3);
                    float s1, c1, s2, c2;
                    __sincosf(B2D_TWO_PI_F * u2, &s1, &c1);
                    __sincosf(B2D_TWO_PI_F * u4, &s2, &c2);
                    eps[4 * c + 0] = m1 * c1; eps[4 * c + 1] = m1 * s1;
                    eps[4 * c + 2] = m2 * c2; eps[4 * c + 3] = m2 * s2;
                }
            }
        }
        float lin = p.lin_b;
#pragma unroll
        for (int h = 0; h < MAXD; ++h) {
            if (h < dim) {
                const float theta = __fadd_rn(__fmul_rn(rad, (float)(h + 1)), __ldg(p.rand_ini + h));   // (:143,146)
                const float sn = sin_reduced(__fmul_rn(B2D_TWO_PI_F, theta));                             // (:147)
                const float v = __fadd_rn(__fmul_rn(sn, samp_uv), __fmul_rn(namp, eps[h]));              // (:159,163-164)
                if (p.merged) lin = fmaf(__ldg(p.lin_w + h), v, lin);                                     // l_linear (:203)
                else row[h] = v;
            }
        }
        if (p.merged) p.merged[(size_t)b * T + t] = tanhf(lin);                                           // l_tanh (:203)
    }
    if (p.merged) return;          // uniform per launch: no tile to write back
    __syncthreads();
    float* dst = p.out + base;
    if ((base & 3) == 0 && (nflat & 3) == 0) {
        for (int i = tid; i < (nflat >> 2); i += kTile)
            b2d::st_global_v4(dst + 4 * i, reinterpret_cast<const float4*>(tile)[i]);
    } else {
        for (int i = tid; i < nflat; i += kTile) dst[i] = tile[i];
    }
}


// ---- v2: four consecutive samples per thread --------------------------------------------------------------
// The kernel is issue-bound, not write-bound (ncu: 81 % issue-active at 23 % of DRAM peak), so v2 removes
// instructions rather than bytes:
//   * 4 samples x DIM harmonics = 4*DIM normals = exactly DIM Philox4x32-10 blocks (v1: ceil(DIM/4) blocks per
//     sample, 12 normals for 9 harmonics); counter = flat quad index, so the stream is still a pure function of
//     (seed, global utterance, position) and independent of how the batch is sharded;
//   * Box-Muller straight on the .ftz approximate units (no denormal fix-up code around the MUFUs), uniforms
//     assembled with integer ops, rint() by the add-magic-constant trick: the SFU pipe only sees 4 MUFU per
//     normal pair and one per sine;
//   * frame lookup, f0/sr, rand_ini and the Linear weights once per thread instead of once per sample;
//   * MODE 1 only: the fp32 chain of two samples at a time as register pairs (mul2 / add2 / fma2 below, scalar
//     instructions on Hopper) -- kept as an option;
//   * FUSED (SourceModuleHnNSF): no shared-memory tile at all, one 128-bit store of 4 merged samples.
constexpr int kQ = 4;
constexpr int kThreads4 = 128;
constexpr int kTile4 = kThreads4 * kQ;

typedef unsigned long long u64;
__device__ __forceinline__ u64 pack2(float lo, float hi) { u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ void unpack2(u64 v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ u64 dup2(float x) { return pack2(x, x); }
// lane-wise pair arithmetic: Hopper has no f32x2 instructions, so each is two scalar ones (the explicit _rn
// intrinsics are never contracted into an FMA)
__device__ __forceinline__ u64 mul2(u64 a, u64 b) {
    float a0, a1, b0, b1; unpack2(a, a0, a1); unpack2(b, b0, b1); return pack2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ u64 add2(u64 a, u64 b) {
    float a0, a1, b0, b1; unpack2(a, a0, a1); unpack2(b, b0, b1); return pack2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
    float a0, a1, b0, b1, c0, c1; unpack2(a, a0, a1); unpack2(b, b0, b1); unpack2(c, c0, c1);
    return pack2(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}
__device__ __forceinline__ float lg2_ftz(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float sin_ftz(float x) { float y; asm("sin.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float cos_ftz(float x) { float y; asm("cos.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

__device__ __forceinline__ float sqrt_ftz(float x) { float y; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

// Four standard normals from one Philox block (Box-Muller, two pairs).  The SFU ("XU") pipe is the scarce unit
// here -- 16 lanes/clk/SM shared by MUFU, FRND and the int->float conversions -- so the uniforms are built with
// integer ops (23 random mantissa bits under exponent 0: f in [1,2)) instead of I2F, and each pair costs exactly
// four MUFU: LG2, SQRT, SIN, COS.
//   radius: u = 2 - f in (0,1] (2^-23 granularity, |z| <= 5.65);  lg2(1) = +0 exactly, so a >= 0 and no clamp
//   angle : sin/cos(2 pi f) = sin/cos(2 pi (f-1)): the whole turn is removed by the SFU's own range reduction
__device__ __forceinline__ void normals4(const uint4 r, float* z) {
    const float f1 = __uint_as_float((r.x >> 9) | 0x3f800000u), f2 = __uint_as_float((r.y >> 9) | 0x3f800000u);
    const float f3 = __uint_as_float((r.z >> 9) | 0x3f800000u), f4 = __uint_as_float((r.w >> 9) | 0x3f800000u);
    const float m1 = sqrt_ftz(lg2_ftz(2.0f - f1) * -1.3862943611198906f);      // sqrt(-2 ln u)
    const float m3 = sqrt_ftz(lg2_ftz(2.0f - f3) * -1.3862943611198906f);
    const float t2 = f2 * B2D_TWO_PI_F, t4 = f4 * B2D_TWO_PI_F;
    z[0] = m1 * cos_ftz(t2); z[1] = m1 * sin_ftz(t2);
    z[2] = m3 * cos_ftz(t4); z[3] = m3 * sin_ftz(t4);
}

// round to nearest integer (ties to even) on the FMA pipe instead of FRND (SFU): valid for |x| < 2^22
#define B2D_RINT_MAGIC 12582912.0f
__device__ __forceinline__ float rint_fma(float x) { return __fsub_rn(__fadd_rn(x, B2D_RINT_MAGIC), B2D_RINT_MAGIC); }

// sin(fl(2 pi theta)) for theta (revolutions) up to a few hundred: k = rint(theta) is the multiple of 2 pi to remove
__device__ __forceinline__ float sin_turns(float theta) {
    const float arg = __fmul_rn(B2D_TWO_PI_F, theta);                                  // (:147) the reference's fp32 argument
    const float k = rint_fma(theta);
    float r = fmaf(k, -6.2831854820251465f, arg);
    r = fmaf(k, 1.7484555e-7f, r);
    return __sinf(r);
}

// MODE 0: scalar arithmetic (default); MODE 1: register-pair arithmetic.
// ROUNDS: Philox rounds of the in-kernel noise (10 standard; 7 = `v2r7`, see b2d_common.cuh)
template <int DIM, bool FUSED, int MODE, int ROUNDS = 10>
__global__ void __launch_bounds__(kThreads4, 6) sinegen4_kernel(SgParams p) {
    extern __shared__ __align__(16) float tile[];  // [kTile4 * DIM]; untouched when FUSED without noise_in
    const int b = blockIdx.y;
    const int T = p.nF * p.upp;
    const int t0 = blockIdx.x * kTile4;
    const int nt = min(kTile4, T - t0);
    const int tid = threadIdx.x;
    const size_t base = ((size_t)b * T + t0) * DIM;
    const int nflat = nt * DIM;
    const bool vec_ok = (base & 3) == 0 && (nflat & 3) == 0;

    if (p.noise_in) {  // stage the noise tile (coalesced)
        const float* src = p.noise_in + base;
        if (vec_ok) {
            for (int i = tid; i < (nflat >> 2); i += kThreads4)
                reinterpret_cast<float4*>(tile)[i] = __ldg(reinterpret_cast<const float4*>(src) + i);
        } else {
            for (int i = tid; i < nflat; i += kThreads4) tile[i] = src[i];
        }
        __syncthreads();
    }

    const int lt = kQ * tid;                        // first local sample of this thread
    float4* rows4 = reinterpret_cast<float4*>(tile + (size_t)lt * DIM);   // kQ*DIM floats = DIM float4, 16-byte aligned
    if (lt < nt) {
        const int tb = t0 + lt;
        const unsigned long long utt = (unsigned long long)(p.utt_off + b);
        const uint32_t q0 = (uint32_t)(tb >> 2) * DIM;          // flat quad index of this thread's first Philox block
        const uint2 key = make_uint2((uint32_t)p.seed, (uint32_t)(p.seed >> 32));
        float eps[kQ * DIM];                        // noise, then overwritten in place by the outputs
        if (p.noise_in) {
#pragma unroll
            for (int c = 0; c < DIM; ++c) {
                const float4 v = rows4[c];
                eps[4 * c] = v.x; eps[4 * c + 1] = v.y; eps[4 * c + 2] = v.z; eps[4 * c + 3] = v.w;
            }
        } else {
#pragma unroll
            for (int c = 0; c < DIM; ++c)
                normals4(b2d::philox4x32<ROUNDS>(make_uint4(q0 + c, 0x51e6e004u, (uint32_t)utt, (uint32_t)(utt >> 32)), key), eps + 4 * c);
        }
        // per-sample frame quantities; consecutive samples share a frame except at a boundary
        int k, j;
        if (p.upp_shift >= 0) { k = tb >> p.upp_shift; j = tb & (p.upp - 1); }
        else { k = tb / p.upp; j = tb - k * p.upp; }
        float s, accp, namp, samp;
        auto load_frame = [&](int kk) {
            const float f = __ldg(p.f0 + (size_t)b * p.nF + kk);
            s = __fdiv_rn(f, p.sr);                                                      // f0 / sr
            accp = __ldg(p.acc_prev + (size_t)b * p.nF + kk);
            const bool voiced = f > p.thr;
            namp = voiced ? p.namp_voiced : p.namp_unvoiced;                             // (:162)
            samp = voiced ? p.sine_amp : 0.0f;      // (sin*sine_amp)*uv == sin*(sine_amp*uv) for uv in {0,1}
        };
        load_frame(k);
        float radv[kQ], nampv[kQ], sampv[kQ];
#pragma unroll
        for (int i = 0; i < kQ; ++i) {
            if (i > 0 && ++j == p.upp) { j = 0; ++k; if (k < p.nF) load_frame(k); }
            radv[i] = __fadd_rn(__fmul_rn(s, (float)(j + 1)), accp);                    // (:138,141)
            nampv[i] = namp; sampv[i] = samp;
        }
        float lin[kQ];
#pragma unroll
        for (int i = 0; i < kQ; ++i) lin[i] = p.lin_b;

        if (MODE == 1) {
            u64 rad2[kQ / 2], namp2[kQ / 2], samp2[kQ / 2];
#pragma unroll
            for (int g = 0; g < kQ / 2; ++g) {
                rad2[g] = pack2(radv[2 * g], radv[2 * g + 1]);
                namp2[g] = pack2(nampv[2 * g], nampv[2 * g + 1]);
                samp2[g] = pack2(sampv[2 * g], sampv[2 * g + 1]);
            }
#pragma unroll
            for (int h = 0; h < DIM; ++h) {
                const float rho = __ldg(p.rand_ini + h);
                const float wh = FUSED ? __ldg(p.lin_w + h) : 0.0f;
#pragma unroll
                for (int g = 0; g < kQ / 2; ++g) {
                    const u64 th = add2(mul2(rad2[g], dup2((float)(h + 1))), dup2(rho));                 // (:143,146)
                    const u64 arg = mul2(th, dup2(B2D_TWO_PI_F));                                           // (:147)
                    const u64 kk = add2(add2(th, dup2(B2D_RINT_MAGIC)), dup2(-B2D_RINT_MAGIC));             // rint, FMA pipe
                    float r0, r1;
                    unpack2(fma2(kk, dup2(1.7484555e-7f), fma2(kk, dup2(-6.2831854820251465f), arg)), r0, r1);
                    const u64 sn = pack2(__sinf(r0), __sinf(r1));
                    const int e0 = (2 * g) * DIM + h, e1 = (2 * g + 1) * DIM + h;
                    float v0, v1;
                    unpack2(add2(mul2(sn, samp2[g]), mul2(namp2[g], pack2(eps[e0], eps[e1]))), v0, v1);  // (:159,163-164)
                    if (FUSED) { lin[2 * g] = fmaf(wh, v0, lin[2 * g]); lin[2 * g + 1] = fmaf(wh, v1, lin[2 * g + 1]); }   // (:203)
                    else { eps[e0] = v0; eps[e1] = v1; }
                }
            }
        } else {
#pragma unroll
            for (int h = 0; h < DIM; ++h) {
                const float rho = __ldg(p.rand_ini + h);
                const float wh = FUSED ? __ldg(p.lin_w + h) : 0.0f;
#pragma unroll
                for (int i = 0; i < kQ; ++i) {
                    const float theta = __fadd_rn(__fmul_rn(radv[i], (float)(h + 1)), rho);              // (:143,146)
                    const float sn = sin_turns(theta);                                                       // (:147)
                    const float v = __fadd_rn(__fmul_rn(sn, sampv[i]), __fmul_rn(nampv[i], eps[i * DIM + h]));   // (:159,163-164)
                    if (FUSED) lin[i] = fmaf(wh, v, lin[i]);                                                 // (:203)
                    else eps[i * DIM + h] = v;
                }
            }
        }

        if (FUSED) {
            float* dst = p.merged + (size_t)b * T + tb;
            if (tb + kQ <= T && ((((size_t)b * T + tb) & 3) == 0)) {
                b2d::st_global_v4(dst, make_float4(tanhf(lin[0]), tanhf(lin[1]), tanhf(lin[2]), tanhf(lin[3])));   // l_tanh (:203)
            } else {
#pragma unroll
                for (int i = 0; i < kQ; ++i) if (tb + i < T) dst[i] = tanhf(lin[i]);
            }
        } else {
#pragma unroll
            for (int c = 0; c < DIM; ++c) rows4[c] = make_float4(eps[4 * c], eps[4 * c + 1], eps[4 * c + 2], eps[4 * c + 3]);
        }
    }
    if (FUSED) return;
    __syncthreads();
    float* dst = p.out + base;
    if (vec_ok) {
        for (int i = tid; i < (nflat >> 2); i += kThreads4)
            b2d::st_global_v4(dst + 4 * i, reinterpret_cast<const float4*>(tile)[i]);
    } else {
        for (int i = tid; i < nflat; i += kThreads4) dst[i] = tile[i];
    }
}

template <int DIM, bool FUSED, int MODE, int ROUNDS = 10>
void launch_v2_as(const SgParams& p, dim3 grid, size_t smem, cudaStream_t st) {
    // 18 KB tiles x 6 resident CTAs: ask for the large shared-memory split (per launch: attributes are per device)
    cudaFuncSetAttribute(sinegen4_kernel<DIM, FUSED, MODE, ROUNDS>, cudaFuncAttributePreferredSharedMemoryCarveout,
                         cudaSharedmemCarveoutMaxShared);
    sinegen4_kernel<DIM, FUSED, MODE, ROUNDS><<<grid, kThreads4, smem, st>>>(p);
}

template <int DIM>
void launch_v2(const SgParams& p, int B, long long T, int impl, cudaStream_t st) {
    const dim3 grid((unsigned)((T + kTile4 - 1) / kTile4), B);
    const bool fused = p.merged != nullptr;
    const size_t smem = (!fused || p.noise_in) ? (size_t)kTile4 * DIM * sizeof(float) : 0;
    if (fused) {
        if (impl == 2) launch_v2_as<DIM, true, 0>(p, grid, smem, st);
        else if (impl == 4) launch_v2_as<DIM, true, 0, 7>(p, grid, smem, st);
        else launch_v2_as<DIM, true, 1>(p, grid, smem, st);
    } else {
        if (impl == 2) launch_v2_as<DIM, false, 0>(p, grid, smem, st);
        else if (impl == 4) launch_v2_as<DIM, false, 0, 7>(p, grid, smem, st);
        else launch_v2_as<DIM, false, 1>(p, grid, smem, st);
    }
}

std::atomic<int> g_sinegen_impl{0};   // 0 auto, 1 v1 (one sample per thread), 2 v2 scalar, 3 v2 register pairs, 4 v2 scalar with Philox-7 noise

}  // namespace

extern "C" int b2d_set_sinegen_impl(int impl) {
    if (impl < 0 || impl > 4) return b2d::fail(B2D_ERR_UNSUPPORTED, "set_sinegen_impl: %d not in 0..4", impl);
    g_sinegen_impl.store(impl, std::memory_order_relaxed);
    return 0;
}

static int sinegen_launch(const float* f0, const float* rand_ini, const float* noise_in, uint64_t seed,
                          int64_t utterance_offset, int B, int n_frames, int upp, int dim, double sampling_rate,
                          float sine_amp, float noise_std, float voiced_threshold, float* acc_workspace, float* out,
                          const float* lin_w, float lin_b, float* merged, void* stream);

extern "C" int b2d_sinegen(const float* f0, const float* rand_ini, const float* noise_in, uint64_t seed,
                           int64_t utterance_offset, int B, int n_frames, int upp, int dim,
                           double sampling_rate, float sine_amp, float noise_std, float voiced_threshold,
                           float* acc_workspace, float* out, void* stream) {
    if (!out) return b2d::fail(B2D_ERR_NULL, "sinegen: null pointer");
    return sinegen_launch(f0, rand_ini, noise_in, seed, utterance_offset, B, n_frames, upp, dim, sampling_rate, sine_amp,
                          noise_std, voiced_threshold, acc_workspace, out, nullptr, 0.f, nullptr, stream);
}

extern "C" int b2d_source_module(const float* f0, const float* rand_ini, const float* noise_in, uint64_t seed,
                                 int64_t utterance_offset, int B, int n_frames, int upp, int dim,
                                 double sampling_rate, float sine_amp, float noise_std, float voiced_threshold,
                                 const float* linear_weight, float linear_bias, float* acc_workspace, float* merged,
                                 void* stream) {
    if (!linear_weight || !merged) return b2d::fail(B2D_ERR_NULL, "source_module: null pointer");
    return sinegen_launch(f0, rand_ini, noise_in, seed, utterance_offset, B, n_frames, upp, dim, sampling_rate, sine_amp,
                          noise_std, voiced_threshold, acc_workspace, nullptr, linear_weight, linear_bias, merged, stream);
}

static int sinegen_launch(const float* f0, const float* rand_ini, const float* noise_in, uint64_t seed,
                          int64_t utterance_offset, int B, int n_frames, int upp, int dim, double sampling_rate,
                          float sine_amp, float noise_std, float voiced_threshold, float* acc_workspace, float* out,
                          const float* lin_w, float lin_b, float* merged, void* stream) {
    if (!f0 || !rand_ini || !acc_workspace) return b2d::fail(B2D_ERR_NULL, "sinegen: null pointer");
    if (B <= 0 || n_frames <= 0 || upp <= 0 || dim <= 0) return b2d::fail(B2D_ERR_SHAPE, "sinegen: bad shape");
    if (dim > kMaxDim) return b2d::fail(B2D_ERR_UNSUPPORTED, "sinegen: dim %d > %d", dim, kMaxDim);
    if (B > 65535) return b2d::fail(B2D_ERR_UNSUPPORTED, "sinegen: batch %d > 65535", B);
    if ((out && !b2d::aligned16(out)) || (noise_in && !b2d::aligned16(noise_in)) || (merged && !b2d::aligned16(merged)))
        return b2d::fail(B2D_ERR_ALIGN, "sinegen: out / merged / noise_in must be 16-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    sinegen_scan_kernel<<<B, kScanThreads, 0, st>>>(f0, n_frames, upp, (float)sampling_rate, acc_workspace);
    int rc = b2d::check_launch("sinegen_scan");
    if (rc) return rc;
    SgParams p;
    p.f0 = f0; p.acc_prev = acc_workspace; p.rand_ini = rand_ini; p.noise_in = noise_in; p.out = out;
    p.nF = n_frames; p.upp = upp; p.dim = dim;
    p.sr = (float)sampling_rate; p.sine_amp = sine_amp; p.thr = voiced_threshold;
    p.upp_shift = -1;
    for (int sft = 0; sft < 30; ++sft) if ((1 << sft) == upp) p.upp_shift = sft;
    // noise_amp = uv*noise_std + (1-uv)*sine_amp/3 in fp32 with the reference's operation order (:162)
    p.namp_voiced = (1.0f * noise_std) + ((0.0f * sine_amp) / 3.0f);
    p.namp_unvoiced = (0.0f * noise_std) + ((1.0f * sine_amp) / 3.0f);
    p.seed = seed; p.utt_off = utterance_offset;
    p.lin_w = lin_w; p.lin_b = lin_b; p.merged = merged;
    const long long T = (long long)n_frames * upp;
    const int sel = g_sinegen_impl.load(std::memory_order_relaxed);
    // auto = four samples per thread, scalar arithmetic, Philox4x32-7 normals (KS / correlation
    // tests in tests/test_gpu_combsub_sinegen.py); 2 selects the same kernel with the standard 10 rounds
    const int impl = sel == 0 ? 4 : sel;
    if (impl >= 2 && (dim == 9 || dim == 1)) {
        if (dim == 9) launch_v2<9>(p, B, T, impl, st);
        else launch_v2<1>(p, B, T, impl, st);
        return b2d::check_launch("sinegen(v2)");
    }
    const dim3 grid((unsigned)((T + kTile - 1) / kTile), B);
    const size_t smem = kTile * dim * sizeof(float);
    if (dim == 9) sinegen_kernel<9><<<grid, kTile, smem, st>>>(p);
    else if (dim == 1) sinegen_kernel<1><<<grid, kTile, smem, st>>>(p);
    else sinegen_kernel<0><<<grid, kTile, smem, st>>>(p);
    return b2d::check_launch("sinegen");
}
