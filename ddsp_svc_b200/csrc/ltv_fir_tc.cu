// K4-TC: the linear time-varying FIR of ltv_fir.cu on the Hopper tensor cores (wgmma tf32,
// accumulators in registers), 3xTF32 split for fp32-level accuracy.
//
// Same tiling and algebra as ltv_fir.cu: a tile is P = 512 consecutive outputs
// n = f P - (L/2+1) + i; per tap segment the inputs are the 2P samples xs[q], q = m - (gP - P), and
//     y[i] = sum_tau' xs[P-1+i-tau'] G[tau'] + ((i-1)/P) sum_tau' xs[P-1+i-tau'] E[tau'],
// where (G,E) are the "A" tables for inputs of frame g (q >= P) and the "B" tables for inputs of
// frame g-1 (q < P).  The table switch depends only on the INPUT sample, so with x+ = xs 1[q>=P],
// x- = xs 1[q<P]:
//     Y = Hankel(x+) . Toep(A tables) + Hankel(x-) . Toep(B tables)
// with  Hankel(x)[r, c] = x[4 r + c]           (128 rows r, i = 4 r + j)
//       Toep(T)[c, (t, j)] = T_t[P-1+j-c]      (t in {G,E}, j = 0..3  ->  N = 8 columns)
// A Hankel matrix with row shift 4 is exactly a K-major, no-swizzle wgmma operand VIEW of the linear
// signal in shared memory (rows 16 B apart, K-chunks 16 B apart: SBO = 128 B, LBO = 16 B -- core
// matrices overlap; the descriptor only describes addresses), so the 512 x 515 operand is never
// materialised.  The small Toeplitz operand (8 x 520) is.
//
// fp32 accuracy: the tensor core truncates fp32 inputs to tf32, so every operand is split with
// round-to-nearest into hi + lo (lo rounded to tf32 as well) and each product is accumulated as
// hi*hi + lo*hi + hi*lo in the fp32 accumulator (3xTF32): relative error ~2^-21 per term,
// i.e. the same level as an fp32 FMA chain over 510 taps.
//
// STATUS: correct (parity tests run it), NOT the default.  Work per (tile, filter, segment) is
// 2 regions x 3 split products x 65 K-steps x 2 row halves = 780 wgmmas of 64x8x8, and each also
// fetches its 64 x 32 B Hankel operand from shared memory: with only N = 8 columns to amortise it the
// kernel is operand-bandwidth bound.  A time-varying FIR is matrix-VECTOR shaped (every (utterance,
// frame) has its own input and its own impulse response), so there is no second large dimension to
// batch along N.  Also note the fp32 tensor-core accumulator truncates: ~5e-6 relative error after 390
// accumulation steps.  Kept as a tested alternative (b2d_set_fir_impl(2)).  One CTA (one warpgroup) per
// (tile, filter): its 128 threads build the operands (tables, hi/lo splits, Toeplitz matrices: ~91 KB
// shared memory -> 2 CTAs per SM, so one CTA's operand build overlaps the other's MMAs), issue the
// wgmmas for rows 0..63 and 64..127 of the tile, stage the accumulators through shared memory, apply
// the (i-1)/P recombination and store float4s.
// `mix` (signal = harmonic + noise) is formed with red.global.add.v4.f32 into a zeroed buffer; with
// exactly two addends the result does not depend on arrival order.
#include "b2d_common.cuh"

namespace {

constexpr int kP = 512;
constexpr int kThreads = 128;
constexpr int kK = kP + 8;            // K extent of the GEMM (515 needed), multiple of 8
constexpr int kSteps = kK / 8;        // 65
constexpr int kXLen = 4 * 127 + kK + 4;   // 1032 floats per Hankel source array
constexpr int kBmat = (kK / 4) * 8 * 4;   // floats per Toeplitz operand: [130 chunks][8 rows][4]

struct TcJob {
    const float* x;   // [B,T] or nullptr -> in-kernel uniform noise
    const float* ir;  // [B,nF,L]
    float* y;         // [B,T] or nullptr
    int L;
};
struct TcParams {
    TcJob job[2];
    const float* addend;  // [B,T] or nullptr (single-job launches only)
    float* mix;           // [B,T] or nullptr
    int mix_atomic;       // 1: accumulate into a zeroed mix with red.add (two jobs)
    unsigned long long seed;
    long long utt_off;
    int nF, T;
};

__device__ __forceinline__ uint32_t tf32_rn_bits(float x) {   // round-to-nearest-even to 10 mantissa bits
    uint32_t u = __float_as_uint(x);
    u += 0x00000FFFu + ((u >> 13) & 1u);
    return u & 0xFFFFE000u;
}
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    hi = __uint_as_float(tf32_rn_bits(x));
    lo = __uint_as_float(tf32_rn_bits(x - hi));
}
// wgmma shared-memory descriptor, K-major, layout type 0 = no swizzle
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}
// D[64 x 8] += A[64 x 8] . B[8 x 8], both tf32 from shared memory
__device__ __forceinline__ void wgmma_tf32_m64n8k8(float (&d)[4], uint64_t da, uint64_t db) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n8k8.f32.tf32.tf32 {%0, %1, %2, %3}, %4, %5, 1, 1, 1;\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "l"(da), "l"(db));
}
__device__ __forceinline__ void fence_reg(float& r) { asm volatile("" : "+f"(r)::"memory"); }
__device__ __forceinline__ void red_add_v4(float* p, float4 v) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// shared memory: xs[4][kXLen] (x+hi, x+lo, x-hi, x-lo) | bm[4][kBmat] (A hi, A lo, B hi, B lo) | tab[4][kP]
// (tab doubles as the [128][8] accumulator staging of the epilogue)
constexpr size_t kSmem = (size_t)(4 * kXLen + 4 * kBmat + 4 * kP) * sizeof(float) + 64;

__global__ void __launch_bounds__(kThreads, 2) ltv_fir_tc_kernel(TcParams p) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float* xs = reinterpret_cast<float*>(smem_raw);     // 4 arrays
    float* bm = xs + 4 * kXLen;                         // 4 Toeplitz operands
    float* tab = bm + 4 * kBmat;                        // GA, EA, GB, EB  [kP] each

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int f = blockIdx.x, b = blockIdx.y, jobi = blockIdx.z;
    TcJob jb;
    jb.x = jobi ? p.job[1].x : p.job[0].x;
    jb.ir = jobi ? p.job[1].ir : p.job[0].ir;
    jb.y = jobi ? p.job[1].y : p.job[0].y;
    jb.L = jobi ? p.job[1].L : p.job[0].L;
    const int L = jb.L, Mh = L / 2 + 1, NS = (L + kP - 1) / kP;
    const int nF = p.nF, T = p.T;
    const float* xrow = jb.x ? jb.x + (size_t)b * T : nullptr;
    const float* irb = jb.ir + (size_t)b * nF * L;
    const float invP = 1.0f / (float)kP;

    // zero the Hankel sources' tails once (q >= 2P are never written)
    for (int i = tid; i < 4 * kXLen; i += kThreads) xs[i] = 0.f;
    __syncthreads();

    float acc[2][4];                                   // rows 0..63 and 64..127 of the tile, N = 8
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[h][i] = 0.f;
    bool any = false;
    for (int s = 0; s < NS; ++s) {
        const int g = f - s;
        if (g < 0 || g > nF) continue;                 // no inputs inside [0,T) for this segment
        if (any) __syncthreads();                      // previous segment's MMAs are done (wait_group): operands may be rebuilt
        // ---- input tile m in [gP-P, gP+P): split into x+ / x- and hi / lo ----
        const int mbase = g * kP - kP;
        for (int c = tid; c < (kP >> 1); c += kThreads) {
            const int q0 = c << 2, m = mbase + q0;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m >= 0 && m < T) {
                if (xrow) v = __ldg(reinterpret_cast<const float4*>(xrow + m));
                else v = b2d::philox_uniform_pm1(p.seed, (unsigned long long)(p.utt_off + b), (uint32_t)(m >> 2));
            }
            float4 hi, lo;
            split_tf32(v.x, hi.x, lo.x); split_tf32(v.y, hi.y, lo.y);
            split_tf32(v.z, hi.z, lo.z); split_tf32(v.w, hi.w, lo.w);
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            const bool plus = q0 >= kP;                // whole quad on one side (P % 4 == 0)
            *reinterpret_cast<float4*>(xs + 0 * kXLen + q0) = plus ? hi : z;
            *reinterpret_cast<float4*>(xs + 1 * kXLen + q0) = plus ? lo : z;
            *reinterpret_cast<float4*>(xs + 2 * kXLen + q0) = plus ? z : hi;
            *reinterpret_cast<float4*>(xs + 3 * kXLen + q0) = plus ? z : lo;
        }
        // ---- tables for taps tau = sP + tau' (same as ltv_fir.cu) ----
        const float* hm = irb + (size_t)min(max(g - 1, 0), nF - 1) * L;
        const float* h0 = irb + (size_t)min(max(g, 0), nF - 1) * L;
        const float* hp = irb + (size_t)min(max(g + 1, 0), nF - 1) * L;
        for (int tp = tid; tp < kP; tp += kThreads) {
            const int tau = s * kP + tp;
            float vm = 0.f, v0 = 0.f, vp = 0.f;
            if (tau < L) { vm = __ldg(hm + tau); v0 = __ldg(h0 + tau); vp = __ldg(hp + tau); }
            const float w = (float)tp * invP;
            const float eA = vp - v0, eB = v0 - vm;
            tab[0 * kP + tp] = fmaf(-w, eA, v0);   // GA
            tab[1 * kP + tp] = eA;                 // EA
            tab[2 * kP + tp] = fmaf(-w, eB, v0);   // GB
            tab[3 * kP + tp] = eB;                 // EB
        }
        __syncthreads();
        // ---- Toeplitz operands: bm[R*2 + {hi,lo}][chunk cc][row n = 4 t + j][e] = T_{R,t}[P-1+j-(4cc+e)] ----
        for (int item = tid; item < 2 * (kK / 4) * 8; item += kThreads) {
            const int R = item / ((kK / 4) * 8);
            const int rem = item - R * ((kK / 4) * 8);
            const int cc = rem >> 3, n = rem & 7;
            const int t = n >> 2, j = n & 3;
            const float* tb = tab + (2 * R + t) * kP;
            float4 hi, lo;
            float v[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int u = kP - 1 + j - (4 * cc + e);
                v[e] = (u >= 0 && u < kP) ? tb[u] : 0.f;
            }
            split_tf32(v[0], hi.x, lo.x); split_tf32(v[1], hi.y, lo.y);
            split_tf32(v[2], hi.z, lo.z); split_tf32(v[3], hi.w, lo.w);
            *reinterpret_cast<float4*>(bm + (2 * R + 0) * kBmat + (cc * 8 + n) * 4) = hi;
            *reinterpret_cast<float4*>(bm + (2 * R + 1) * kBmat + (cc * 8 + n) * 4) = lo;
        }
        b2d::fence_proxy_async();                      // generic-proxy writes -> visible to the tensor core
        __syncthreads();
        // ---- MMAs: regions (x+, A tables), (x-, B tables); products hi*hi, lo*hi, hi*lo ----
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 4; ++i) fence_reg(acc[h][i]);
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
        {
            const uint32_t xs_a = b2d::smem_u32(xs), bm_a = b2d::smem_u32(bm);
#pragma unroll 1
            for (int R = 0; R < 2; ++R) {
#pragma unroll 1
                for (int pr = 0; pr < 3; ++pr) {
                    const int xi = 2 * R + (pr == 1 ? 1 : 0);          // x hi, lo, hi
                    const int bi = 2 * R + (pr == 2 ? 1 : 0);          // T hi, hi, lo
                    // Hankel view: rows 16 B apart (8-row blocks 128 B), K chunks 16 B apart; K-step = 32 B;
                    // rows 64..127 start 64 x 16 B later
                    uint64_t da = make_desc(xs_a + xi * kXLen * 4, 16, 128);
                    // Toeplitz operand: [chunk][8 rows][4]: chunks 128 B apart; K-step = 2 chunks = 256 B
                    uint64_t db = make_desc(bm_a + bi * kBmat * 4, 128, 128);
#pragma unroll 5
                    for (int ks = 0; ks < kSteps; ++ks) {
                        wgmma_tf32_m64n8k8(acc[0], da, db);
                        wgmma_tf32_m64n8k8(acc[1], da + 64, db);
                        da += 2;     // +32 B  (start address field is in 16-byte units)
                        db += 16;    // +256 B
                    }
                }
            }
        }
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 4; ++i) fence_reg(acc[h][i]);
        any = true;
    }

    // ---- epilogue: registers -> [128][8] staging -> y = acc1 + ((i-1)/P) acc2 ----
    // accumulator fragment: acc[h][i] is row 64 h + 16 warp + lane / 4 + 8 (i >> 1), column 2 (lane % 4) + (i & 1)
    float4 yv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (any) {
        __syncthreads();                               // every thread is done with tab
        float* stg = tab;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 4; ++i)
                stg[(64 * h + 16 * warp + (lane >> 2) + 8 * (i >> 1)) * 8 + 2 * (lane & 3) + (i & 1)] = acc[h][i];
        __syncthreads();
        float v[8];
#pragma unroll
        for (int c = 0; c < 8; ++c) v[c] = stg[tid * 8 + c];
        const float i0m1 = (float)(4 * tid - 1);
        yv.x = fmaf((i0m1 + 0.f) * invP, v[4], v[0]);
        yv.y = fmaf((i0m1 + 1.f) * invP, v[5], v[1]);
        yv.z = fmaf((i0m1 + 2.f) * invP, v[6], v[2]);
        yv.w = fmaf((i0m1 + 3.f) * invP, v[7], v[3]);
    }
    const int n0 = f * kP - Mh + 4 * tid;
    const bool vec_ok = ((n0 & 3) == 0) && n0 >= 0 && (n0 + 4) <= T;
    const float yy[4] = {yv.x, yv.y, yv.z, yv.w};
    if (jb.y) {
        float* yrow = jb.y + (size_t)b * T;
        if (vec_ok) b2d::st_global_v4(yrow + n0, yv);
        else {
#pragma unroll
            for (int e = 0; e < 4; ++e) if (n0 + e >= 0 && n0 + e < T) yrow[n0 + e] = yy[e];
        }
    }
    if (p.mix) {
        float* mrow = p.mix + (size_t)b * T;
        if (p.mix_atomic) {
            if (vec_ok) red_add_v4(mrow + n0, yv);
            else {
#pragma unroll
                for (int e = 0; e < 4; ++e) if (n0 + e >= 0 && n0 + e < T) atomicAdd(mrow + n0 + e, yy[e]);
            }
        } else {
            const float* arow = p.addend ? p.addend + (size_t)b * T : nullptr;
            if (vec_ok) {
                float4 o = yv;
                if (arow) { const float4 a = __ldg(reinterpret_cast<const float4*>(arow + n0)); o.x += a.x; o.y += a.y; o.z += a.z; o.w += a.w; }
                b2d::st_global_v4(mrow + n0, o);
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    if (n0 + e >= 0 && n0 + e < T) mrow[n0 + e] = yy[e] + (arow ? arow[n0 + e] : 0.f);
            }
        }
    }
}

}  // namespace

namespace b2d {

// Tensor-core path of ltv_fir_launch; same contract.  Requires block size 512.
int ltv_fir_tc_launch(const float* x1, const float* ir1, int taps1, float* y1, const float* x2, const float* ir2,
                      int taps2, float* y2, const float* addend, float* mix, uint64_t seed, int64_t utt_off, int B,
                      int nF, int P, cudaStream_t st) {
    if (P != kP) return fail(B2D_ERR_UNSUPPORTED, "ltv_fir_tc: block size must be 512");
    const int njobs = ir2 ? 2 : 1;
    if (njobs == 2 && (taps1 != taps2 || addend))
        return fail(B2D_ERR_UNSUPPORTED, "ltv_fir_tc: two jobs need equal tap counts and no addend");
    TcParams p;
    p.job[0] = {x1, ir1, y1, taps1};
    p.job[1] = {x2, ir2, y2, njobs == 2 ? taps2 : taps1};
    p.addend = addend;
    p.mix = mix;
    p.mix_atomic = (mix && njobs == 2) ? 1 : 0;
    p.seed = seed; p.utt_off = utt_off; p.nF = nF; p.T = nF * P;
    if (p.mix_atomic) {
        cudaError_t e = cudaMemsetAsync(mix, 0, (size_t)B * nF * P * sizeof(float), st);
        if (e != cudaSuccess) return fail((int)e, "ltv_fir_tc: memset: %s", cudaGetErrorString(e));
    }
    const int Mh = taps1 / 2 + 1;
    const int ntiles = nF + (Mh + P - 1) / P;
    cudaError_t e = cudaFuncSetAttribute(ltv_fir_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem);
    if (e != cudaSuccess) return fail((int)e, "ltv_fir_tc: smem attr: %s", cudaGetErrorString(e));
    cudaFuncSetAttribute(ltv_fir_tc_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    ltv_fir_tc_kernel<<<dim3(ntiles, B, njobs), kThreads, kSmem, st>>>(p);
    return check_launch("ltv_fir_tc");
}

}  // namespace b2d
