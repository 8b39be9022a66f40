// K4: linear time-varying FIR  (reference ddsp/core.py:120-182, fft_convolve).
//
//   y[n] = sum_tau ((1-phi_m) h_f[tau] + phi_m h_{f+1}[tau]) x[m],   m = n + L/2 - tau,
//   f = floor(m/P), phi_m = (m mod P)/P, h_{nF} := h_{nF-1}, x = 0 outside [0,T)
//
// (the reference's Bartlett-windowed 50%-overlap FFT overlap-add is exactly this linear
// interpolation of the per-frame impulse responses along the INPUT index m; only the
// linear-convolution result is reproduced, not its 1533-point FFT).
//
// Tiling.  A CTA computes P consecutive outputs n = f P - (L/2+1) + i, i in [0,P).  The tap
// range is cut into segments of P taps; for segment s the inputs are m = g P - 1 + i - tau'
// with g = f - s, tau' in [0,P): they span exactly the two frames g-1 and g, the switch being
// at tau' = i.  Writing the interpolation weight as (i-1-tau')/P = (i-1)/P - tau'/P,
//
//   y[i] += sum_tau' x[m] G[tau'] + ((i-1)/P) sum_tau' x[m] E[tau'],
//   (G,E) = (h_g - (tau'/P) D_g,     D_g = h_{g+1} - h_g)     for tau' <  i   ("A" tables)
//         = (h_g - (tau'/P) D_{g-1}, D_{g-1} = h_g - h_{g-1}) for tau' >= i   ("B" tables)
//
// so each (output, tap) pair costs exactly 2 FMAs on ONE input sample and two small per-tile
// tables that are built once in shared memory.  A thread owns 8 consecutive outputs and slides
// a 12-sample register window over the input (one 128-bit shared load per 4 taps, XOR-swizzled
// so the stride-8 lane pattern is conflict-free); the table entries are warp-broadcast 128-bit
// loads.  Lanes switch from the A to the B tables at different taps, so the loop body is kept
// uniform (pointer select per step) and the <8-tap band where a thread's outputs straddle the
// switch is fixed up afterwards.  Per 4 taps and thread: 64 FFMA, 3 LDS.128, ~8 integer ops.
//
// Two filters ("jobs") with the same tap count can run in one CTA (Sins: harmonic all-pass and
// noise filter); their outputs are summed through shared memory into `mix` (+ an optional
// addend), so signal = harmonic + noise (ddsp/vocoder.py:609) needs no extra pass.
// White noise input is generated in-kernel (Philox4x32-10) when the job has no input pointer.
#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "b2d_common.cuh"

namespace {

struct FirJob {
    const float* x;   // [B,T] or nullptr -> in-kernel uniform noise
    const float* ir;  // [B,nF,L]
    float* y;         // [B,T] or nullptr
    int L;
};

struct FirParams {
    FirJob job[2];
    int njobs;
    const float* addend;  // [B,T] or nullptr
    float* mix;           // [B,T] or nullptr
    unsigned long long seed;
    long long utt_off;
    int nF, P, T;
};

// Input tile layout: the 2P samples are split into 16-byte chunks; even chunks live in `xe`, odd
// chunks in `xo` (each P/4 float4).  A thread's window advances by one chunk per 4-tap step and
// lanes are 2 chunks apart, so within one load instruction all lanes hit the SAME array at
// consecutive float4 slots: conflict-free without any swizzle arithmetic, and with the loop
// unrolled by 6 (3-register window rotation x even/odd alternation) every address is
// pointer + immediate.
__device__ __forceinline__ float x_at(const float4* xe, const float4* xo, int q) {
    const int c = q >> 2;
    const float4* arr = (c & 1) ? xo : xe;
    return reinterpret_cast<const float*>(arr + (c >> 1))[q & 3];
}

__device__ __forceinline__ void fir_step(const float4& lo, const float4& mid, const float4& hi, const float4& t0,
                                         const float4& t1, float (&a1)[8], float (&a2)[8]) {
    const float W[12] = {lo.x, lo.y, lo.z, lo.w, mid.x, mid.y, mid.z, mid.w, hi.x, hi.y, hi.z, hi.w};
    const float G[4] = {t0.x, t0.z, t1.x, t1.z};
    const float E[4] = {t0.y, t0.w, t1.y, t1.w};
#pragma unroll
    for (int tt = 0; tt < 4; ++tt) {
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            const float xv = W[3 + r - tt];
            a1[r] = fmaf(xv, G[tt], a1[r]);
            a2[r] = fmaf(xv, E[tt], a2[r]);
        }
    }
}

// named barrier per job.  The id must be an immediate: with a register id ptxas reserves all 16
// hardware barriers for the CTA, which caps residency at 4 CTAs/SM (measured).
__device__ __forceinline__ void job_barrier(int job, int nthreads) {
    if (job == 0) asm volatile("bar.sync 1, %0;" ::"r"(nthreads) : "memory");
    else asm volatile("bar.sync 2, %0;" ::"r"(nthreads) : "memory");
}

// threads per job = P/8.  smem per job: xe[P] + xo[P] + tabA[2P] + pad[8] + tabB[2P]; then ybuf[2][P].
template <int MAXT, int MINB>
__global__ void __launch_bounds__(MAXT, MINB) ltv_fir_kernel(FirParams p) {
    extern __shared__ __align__(16) float sm[];
    const int P = p.P, T = p.T, nF = p.nF;
    const int TPJ = P >> 3;
    const int job = threadIdx.x / TPJ;
    const int lt = threadIdx.x - job * TPJ;
    const int b = blockIdx.y, f = blockIdx.x;
    const int per_job = 6 * P + 8;
    float* xs = sm + job * per_job;
    float4* xe = reinterpret_cast<float4*>(xs);
    float4* xo = reinterpret_cast<float4*>(xs + P);
    float* tabA = xs + 2 * P;
    float* tabB = tabA + 2 * P + 8;
    float* ybuf = sm + p.njobs * per_job;  // [njobs][P]

    FirJob jb;  // select by value: dynamic indexing of kernel params would spill them to local memory
    jb.x = job ? p.job[1].x : p.job[0].x;
    jb.ir = job ? p.job[1].ir : p.job[0].ir;
    jb.y = job ? p.job[1].y : p.job[0].y;
    jb.L = job ? p.job[1].L : p.job[0].L;
    const int L = jb.L, Mh = L / 2 + 1;
    const int NS = (L + P - 1) / P;
    const int i0 = lt << 3;
    const float invP = 1.0f / (float)P;
    const float* xrow = jb.x ? jb.x + (size_t)b * T : nullptr;
    const float* irb = jb.ir + (size_t)b * nF * L;

    float a1[8], a2[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) a1[r] = a2[r] = 0.f;

    for (int s = 0; s < NS; ++s) {
        const int g = f - s;
        if (g < 0 || g > nF) continue;  // all inputs of this segment are outside [0,T)
        job_barrier(job, TPJ);          // previous segment's readers are done
        // ---- input tile m in [gP-P, gP+P) -> xs (swizzled) ----
        const int mbase = g * P - P;
        for (int c = lt; c < (P >> 1); c += TPJ) {
            const int m = mbase + (c << 2);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m >= 0 && m < T) {  // T and m are multiples of 4: whole quad in range
                if (xrow) v = __ldg(reinterpret_cast<const float4*>(xrow + m));
                else v = b2d::philox_uniform_pm1(p.seed, (unsigned long long)(p.utt_off + b), (uint32_t)(m >> 2));
            }
            ((c & 1) ? xo : xe)[c >> 1] = v;
        }
        // ---- tables for taps tau = sP + tau' ----
        const float* hm = irb + (size_t)min(max(g - 1, 0), nF - 1) * L;
        const float* h0 = irb + (size_t)min(max(g, 0), nF - 1) * L;
        const float* hp = irb + (size_t)min(max(g + 1, 0), nF - 1) * L;
        for (int tp = lt; tp < P; tp += TPJ) {
            const int tau = s * P + tp;
            float vm = 0.f, v0 = 0.f, vp = 0.f;
            if (tau < L) { vm = __ldg(hm + tau); v0 = __ldg(h0 + tau); vp = __ldg(hp + tau); }
            const float w = (float)tp * invP;
            const float eA = vp - v0, eB = v0 - vm;
            reinterpret_cast<float2*>(tabA)[tp] = make_float2(fmaf(-w, eA, v0), eA);
            reinterpret_cast<float2*>(tabB)[tp] = make_float2(fmaf(-w, eB, v0), eB);
        }
        job_barrier(job, TPJ);

        // ---- main loop: P/4 steps of 4 taps ----
        // step s loads chunk c0 - s with c0 = P/4 - 1 + 2 lt (odd): even steps read xo[k0 - s/2],
        // odd steps read xe[k0 - (s-1)/2], k0 = P/8 - 1 + lt.
        const float4* tA = reinterpret_cast<const float4*>(tabA);
        const float4* tB = reinterpret_cast<const float4*>(tabB);
        const int sw = lt << 1;  // steps < sw use the A tables (tau0 < i0)
        const int nsteps = P >> 2;
        const float4* po = xo + ((P >> 3) - 1 + lt);
        const float4* pe = xe + ((P >> 3) - 1 + lt);
        float4 A = pe[1], Bv = po[1], C;  // chunks c0+1 (even) and c0+2 (odd)
        int step = 0;
#define B2D_FIR_STEP(NEW, MID, HI, SRC, J)                                   \
        {                                                                    \
            const float4* tp4 = ((step + (J)) < sw ? tA : tB) + 2 * (step + (J)); \
            const float4 t0 = tp4[0], t1 = tp4[1];                           \
            NEW = (SRC);                                                     \
            fir_step(NEW, MID, HI, t0, t1, a1, a2);                          \
        }
        for (; step + 6 <= nsteps; step += 6) {
            B2D_FIR_STEP(C, A, Bv, po[0], 0)
            B2D_FIR_STEP(Bv, C, A, pe[0], 1)
            B2D_FIR_STEP(A, Bv, C, po[-1], 2)
            B2D_FIR_STEP(C, A, Bv, pe[-1], 3)
            B2D_FIR_STEP(Bv, C, A, po[-2], 4)
            B2D_FIR_STEP(A, Bv, C, pe[-2], 5)
            po -= 3;
            pe -= 3;
        }
        // remainder (nsteps mod 6 is even because nsteps is a multiple of 64): generic steps
        for (; step < nsteps; step += 2) {
            B2D_FIR_STEP(C, A, Bv, po[0], 0)
            Bv = A; A = C;                       // window: (new, mid, hi) -> (mid, hi) of next step
            B2D_FIR_STEP(C, A, Bv, pe[0], 1)
            Bv = A; A = C;
            po -= 1;
            pe -= 1;
        }
#undef B2D_FIR_STEP
        // ---- band fix-up: taps tau' in [i0, i0+r) belong to the A tables for output r ----
#pragma unroll
        for (int bb = 0; bb < 7; ++bb) {
            const int tp = i0 + bb;
            const float dG = tabA[2 * tp] - tabB[2 * tp];
            const float dE = tabA[2 * tp + 1] - tabB[2 * tp + 1];
#pragma unroll
            for (int r = bb + 1; r < 8; ++r) {
                const float xv = x_at(xe, xo, P - 1 + r - bb);
                a1[r] = fmaf(xv, dG, a1[r]);
                a2[r] = fmaf(xv, dE, a2[r]);
            }
        }
    }

    // ---- combine, store, mix ----
    float yv[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) yv[r] = fmaf((float)(i0 + r - 1) * invP, a2[r], a1[r]);

    const int n0 = f * P - Mh + i0;
    const bool vec_ok = ((n0 & 3) == 0) && n0 >= 0 && (n0 + 8) <= T;
    if (jb.y) {
        float* yrow = jb.y + (size_t)b * T;
        if (vec_ok) {
            b2d::st_global_v4(yrow + n0, make_float4(yv[0], yv[1], yv[2], yv[3]));
            b2d::st_global_v4(yrow + n0 + 4, make_float4(yv[4], yv[5], yv[6], yv[7]));
        } else {
#pragma unroll
            for (int r = 0; r < 8; ++r)
                if (n0 + r >= 0 && n0 + r < T) yrow[n0 + r] = yv[r];
        }
    }
    if (p.mix) {
        if (p.njobs > 1) {
#pragma unroll
            for (int r = 0; r < 8; ++r) ybuf[job * P + i0 + r] = yv[r];
            __syncthreads();
        }
        if (job == 0) {
            float* mrow = p.mix + (size_t)b * T;
            const float* arow = p.addend ? p.addend + (size_t)b * T : nullptr;
#pragma unroll
            for (int r = 0; r < 8; ++r) {
                float v = yv[r];
                if (p.njobs > 1) v += ybuf[P + i0 + r];
                if (arow && n0 + r >= 0 && n0 + r < T) v += arow[n0 + r];
                yv[r] = v;
            }
            if (vec_ok) {
                b2d::st_global_v4(mrow + n0, make_float4(yv[0], yv[1], yv[2], yv[3]));
                b2d::st_global_v4(mrow + n0 + 4, make_float4(yv[4], yv[5], yv[6], yv[7]));
            } else {
#pragma unroll
                for (int r = 0; r < 8; ++r)
                    if (n0 + r >= 0 && n0 + r < T) mrow[n0 + r] = yv[r];
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Variant with 16 outputs per thread and register-pair FMAs (ffma2: two FFMAs on Hopper).  Here the
// accumulators are (a1[r], a2[r]) pairs, the table entries (G, E) pairs straight from LDS.128, and
// each input value is duplicated into a pair once per step; 16 outputs per thread halve the shared
// loads per FMA.  One warp per filter (32 threads x 16 outputs = P = 512), window of 5 chunks
// rotated over a 5-step unrolled loop, inputs in a (chunk ^ (chunk>>3 & 3)) swizzle so the
// stride-4-chunk lane pattern is conflict free.
typedef unsigned long long u64;
__device__ __forceinline__ u64 pack2(float lo, float hi) { u64 r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ void unpack2(u64 v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ void ffma2(u64& d, u64 a, u64 b) {   // lane-wise: two FFMAs on Hopper
    float a0, a1, b0, b1, d0, d1;
    unpack2(a, a0, a1); unpack2(b, b0, b1); unpack2(d, d0, d1);
    d = pack2(fmaf(a0, b0, d0), fmaf(a1, b1, d1));
}

__device__ __forceinline__ int swz4(int c) { return c ^ ((c >> 3) & 3); }

// one 4-tap step; ROT: physical slot of logical chunk L is (L + ROT) % 5, the new (lowest) chunk is logical 0
template <int ROT>
__device__ __forceinline__ void fir16_step(u64 (&ch)[5][4], const float4& xn, const float4& t0, const float4& t1,
                                           u64 (&acc)[16]) {
    constexpr int p0 = ROT % 5;
    ch[p0][0] = pack2(xn.x, xn.x); ch[p0][1] = pack2(xn.y, xn.y);
    ch[p0][2] = pack2(xn.z, xn.z); ch[p0][3] = pack2(xn.w, xn.w);
    const u64 ge[4] = {pack2(t0.x, t0.y), pack2(t0.z, t0.w), pack2(t1.x, t1.y), pack2(t1.z, t1.w)};
#pragma unroll
    for (int tt = 0; tt < 4; ++tt) {
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const int j = 3 + r - tt;                       // window index 0..18
            ffma2(acc[r], ch[((j >> 2) + ROT) % 5][j & 3], ge[tt]);
        }
    }
}

// threads per job = P/16 (a multiple of 32).  smem per job as in ltv_fir_kernel (xs[2P] swizzled here).
template <int MAXT, int MINB>
__global__ void __launch_bounds__(MAXT, MINB) ltv_fir16_kernel(FirParams p) {
    extern __shared__ __align__(16) float sm[];
    const int P = p.P, T = p.T, nF = p.nF;
    const int TPJ = P >> 4;
    const int job = threadIdx.x / TPJ;
    const int lt = threadIdx.x - job * TPJ;
    const int b = blockIdx.y, f = blockIdx.x;
    const int per_job = 6 * P + 8 + (P + (P >> 4) + 8);
    float* xs = sm + job * per_job;
    float4* xs4 = reinterpret_cast<float4*>(xs);
    float* tabA = xs + 2 * P;
    float* tabB = tabA + 2 * P + 8;
    // second difference across frames d2[tp] = h_{g+1} - 2 h_g + h_{g-1}: (GA-GB, EA-EB) = (-w d2, d2) for the
    // band fix-up; padded by one float per 16 taps so the stride-16 lane pattern is conflict free
    float* d2s = tabB + 2 * P;
    float4* ybuf4 = reinterpret_cast<float4*>(sm + p.njobs * per_job);  // [njobs][P/4] float4, swizzled

    FirJob jb;
    jb.x = job ? p.job[1].x : p.job[0].x;
    jb.ir = job ? p.job[1].ir : p.job[0].ir;
    jb.y = job ? p.job[1].y : p.job[0].y;
    jb.L = job ? p.job[1].L : p.job[0].L;
    const int L = jb.L, Mh = L / 2 + 1;
    const int NS = (L + P - 1) / P;
    const int i0 = lt << 4;
    const float invP = 1.0f / (float)P;
    const float* xrow = jb.x ? jb.x + (size_t)b * T : nullptr;
    const float* irb = jb.ir + (size_t)b * nF * L;

    u64 acc[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) acc[r] = 0ull;

    for (int s = 0; s < NS; ++s) {
        const int g = f - s;
        if (g < 0 || g > nF) continue;
        job_barrier(job, TPJ);
        const int mbase = g * P - P;
        for (int c = lt; c < (P >> 1); c += TPJ) {
            const int m = mbase + (c << 2);
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m >= 0 && m < T) {
                if (xrow) v = __ldg(reinterpret_cast<const float4*>(xrow + m));
                else v = b2d::philox_uniform_pm1(p.seed, (unsigned long long)(p.utt_off + b), (uint32_t)(m >> 2));
            }
            xs4[swz4(c)] = v;
        }
        const float* hm = irb + (size_t)min(max(g - 1, 0), nF - 1) * L;
        const float* h0 = irb + (size_t)min(max(g, 0), nF - 1) * L;
        const float* hp = irb + (size_t)min(max(g + 1, 0), nF - 1) * L;
        for (int tp = lt; tp < P; tp += TPJ) {
            const int tau = s * P + tp;
            float vm = 0.f, v0 = 0.f, vp = 0.f;
            if (tau < L) { vm = __ldg(hm + tau); v0 = __ldg(h0 + tau); vp = __ldg(hp + tau); }
            const float w = (float)tp * invP;
            const float eA = vp - v0, eB = v0 - vm;
            reinterpret_cast<float2*>(tabA)[tp] = make_float2(fmaf(-w, eA, v0), eA);
            reinterpret_cast<float2*>(tabB)[tp] = make_float2(fmaf(-w, eB, v0), eB);
            d2s[tp + (tp >> 4)] = eA - eB;
        }
        job_barrier(job, TPJ);

        const float4* tA = reinterpret_cast<const float4*>(tabA);
        const float4* tB = reinterpret_cast<const float4*>(tabB);
        const int c0 = (P >> 2) - 1 + (lt << 2);  // chunk of logical q = P-4+i0 (step 0's new chunk)
        const int sw = lt << 2;                   // steps < sw use the A tables (tau0 < i0)
        const int nsteps = P >> 2;
        u64 ch[5][4];
        // logical chunks 1..4 before step 0 (logical L holds chunk c0 + L) -> physical slots 1..4 (ROT = 0)
#pragma unroll
        for (int Lc = 1; Lc < 5; ++Lc) {
            const float4 v = xs4[swz4(c0 + Lc)];
            ch[Lc][0] = pack2(v.x, v.x); ch[Lc][1] = pack2(v.y, v.y); ch[Lc][2] = pack2(v.z, v.z); ch[Lc][3] = pack2(v.w, v.w);
        }
#define B2D_FIR16_STEP(ROT, J)                                                        \
        {                                                                             \
            const float4* tp4 = ((step + (J)) < sw ? tA : tB) + 2 * (step + (J));     \
            const float4 t0 = tp4[0], t1 = tp4[1];                                    \
            const float4 xn = xs4[swz4(c0 - step - (J))];                             \
            fir16_step<ROT>(ch, xn, t0, t1, acc);                                     \
        }
        int step = 0;
        for (; step + 5 <= nsteps; step += 5) {
            B2D_FIR16_STEP(0, 0)
            B2D_FIR16_STEP(4, 1)
            B2D_FIR16_STEP(3, 2)
            B2D_FIR16_STEP(2, 3)
            B2D_FIR16_STEP(1, 4)
        }
        // remainder (nsteps mod 5 in 0..4): the rotation continues 0, 4, 3, 2 from the loop's end state
        if (step < nsteps) { B2D_FIR16_STEP(0, 0) }
        if (step + 1 < nsteps) { B2D_FIR16_STEP(4, 1) }
        if (step + 2 < nsteps) { B2D_FIR16_STEP(3, 2) }
        if (step + 3 < nsteps) { B2D_FIR16_STEP(2, 3) }
#undef B2D_FIR16_STEP
        // ---- band fix-up: taps tau' in [i0, i0+r) belong to the A tables for output r ----
#pragma unroll
        for (int bb = 0; bb < 15; ++bb) {
            const int tp = i0 + bb;
            const float d2 = d2s[tp + (tp >> 4)];
            const u64 dge = pack2(-((float)tp * invP) * d2, d2);
#pragma unroll
            for (int r = bb + 1; r < 16; ++r) {
                const int q = P - 1 + r - bb;
                const float xv = xs[(swz4(q >> 2) << 2) | (q & 3)];
                ffma2(acc[r], pack2(xv, xv), dge);
            }
        }
    }

    float yv[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) {
        float a1, a2;
        unpack2(acc[r], a1, a2);
        yv[r] = fmaf((float)(i0 + r - 1) * invP, a2, a1);
    }
    const int n0 = f * P - Mh + i0;
    const bool vec_ok = ((n0 & 3) == 0) && n0 >= 0 && (n0 + 16) <= T;
    if (jb.y) {
        float* yrow = jb.y + (size_t)b * T;
        if (vec_ok) {
#pragma unroll
            for (int v4 = 0; v4 < 4; ++v4)
                b2d::st_global_v4(yrow + n0 + 4 * v4, make_float4(yv[4 * v4], yv[4 * v4 + 1], yv[4 * v4 + 2], yv[4 * v4 + 3]));
        } else {
#pragma unroll
            for (int r = 0; r < 16; ++r)
                if (n0 + r >= 0 && n0 + r < T) yrow[n0 + r] = yv[r];
        }
    }
    if (p.mix) {
        if (p.njobs > 1) {
            if (job == 1) {
#pragma unroll
                for (int v4 = 0; v4 < 4; ++v4)
                    ybuf4[swz4((lt << 2) + v4)] = make_float4(yv[4 * v4], yv[4 * v4 + 1], yv[4 * v4 + 2], yv[4 * v4 + 3]);
            }
            __syncthreads();
        }
        if (job == 0) {
            float* mrow = p.mix + (size_t)b * T;
            const float* arow = p.addend ? p.addend + (size_t)b * T : nullptr;
            if (p.njobs > 1) {
#pragma unroll
                for (int v4 = 0; v4 < 4; ++v4) {
                    const float4 o = ybuf4[swz4((lt << 2) + v4)];
                    yv[4 * v4] += o.x; yv[4 * v4 + 1] += o.y; yv[4 * v4 + 2] += o.z; yv[4 * v4 + 3] += o.w;
                }
            }
            if (arow) {
#pragma unroll
                for (int r = 0; r < 16; ++r)
                    if (n0 + r >= 0 && n0 + r < T) yv[r] += arow[n0 + r];
            }
            if (vec_ok) {
#pragma unroll
                for (int v4 = 0; v4 < 4; ++v4)
                    b2d::st_global_v4(mrow + n0 + 4 * v4, make_float4(yv[4 * v4], yv[4 * v4 + 1], yv[4 * v4 + 2], yv[4 * v4 + 3]));
            } else {
#pragma unroll
                for (int r = 0; r < 16; ++r)
                    if (n0 + r >= 0 && n0 + r < T) mrow[n0 + r] = yv[r];
            }
        }
    }
}

// One thread per output sample, straight from the definition.  Any P / L.
__global__ void ltv_fir_generic_kernel(const float* __restrict__ x, const float* __restrict__ ir, int L,
                                       float* __restrict__ y, int nF, int P, int T) {
    const int b = blockIdx.y;
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= T) return;
    const float* xr = x + (size_t)b * T;
    const float* irb = ir + (size_t)b * nF * L;
    const float invP = 1.0f / (float)P;
    float acc = 0.f;
    for (int tau = 0; tau < L; ++tau) {
        const int m = n + L / 2 - tau;
        if (m < 0 || m >= T) continue;
        const int fr = m / P;
        const float phi = (float)(m - fr * P) * invP;
        const float ha = irb[(size_t)fr * L + tau];
        const float hb = irb[(size_t)min(fr + 1, nF - 1) * L + tau];
        acc = fmaf(xr[m], fmaf(phi, hb - ha, ha), acc);
    }
    y[(size_t)b * T + n] = acc;
}

}  // namespace

namespace b2d {

int ltv_fir_tc_launch(const float* x1, const float* ir1, int taps1, float* y1, const float* x2, const float* ir2,
                      int taps2, float* y2, const float* addend, float* mix, uint64_t seed, int64_t utt_off, int B,
                      int nF, int P, cudaStream_t st);
// FFT-domain evaluation (ltv_fir_fft.cu): block size 512, at most 1024 taps per job
bool ltv_fir_fft_supported(int P, int taps1, int taps2, int njobs);
int ltv_fir_fft_launch(const float* x1, const float* ir1, int taps1, float* y1, const float* x2, const float* ir2,
                       int taps2, float* y2, const float* addend, float* mix, uint64_t seed, int64_t utt_off, int B,
                       int nF, int P, cudaStream_t st);

// 0 = auto (FFT-domain kernel where it applies, else CUDA cores), 1 = CUDA-core kernel, 2 = tensor-core kernel
// (block size 512 only), 4 = FFT-domain kernel where it applies (block size 512, <= 1024 taps; other shapes fall
// through to the CUDA-core kernel).   The tensor-core kernel is
// operand-bandwidth bound: with N = 8 columns every MMA re-reads its Hankel operand from shared memory.
static std::atomic<int> g_fir_impl{0};
// CUDA-core variant: 0 = auto (16 outputs/thread + register pairs when the block size is a multiple of 512), 1 = 8 outputs/thread scalar
static std::atomic<int> g_fir_variant{0};

// what "auto" means: the FFT-domain kernel wherever it applies (block size 512, <= 1024 taps), the CUDA-core kernel
// otherwise.
// B2D_FIR_AUTO=cuda in the environment restores the direct form as the automatic choice (A/B runs of whole programs).
static int fir_auto_impl() {
    static const int v = [] {
        const char* e = getenv("B2D_FIR_AUTO");
        return (e && (!strcmp(e, "cuda") || !strcmp(e, "1"))) ? 1 : 4;
    }();
    return v;
}

// true when the FFT-domain kernel is what ltv_fir_launch would pick (the Sins driver then may use its fused variant)
bool fir_fft_selected() {
    const int sel = g_fir_impl.load(std::memory_order_relaxed);
    return (sel == 0 ? fir_auto_impl() : sel) == 4;
}

// internal entry (also used by the CombSub driver): mix = y1 (+ y2) (+ addend)
int ltv_fir_launch(const float* x1, const float* ir1, int taps1, float* y1, const float* x2, const float* ir2,
                   int taps2, float* y2, const float* addend, float* mix, uint64_t seed, int64_t utt_off, int B,
                   int nF, int P, cudaStream_t st) {
    if (!ir1) return fail(B2D_ERR_NULL, "ltv_fir: ir1 is null");
    if (B <= 0 || nF <= 0 || P <= 0 || taps1 <= 0 || (taps1 & 1)) return fail(B2D_ERR_SHAPE, "ltv_fir: bad shape");
    if (P % 256 != 0 || P > 2048)
        return fail(B2D_ERR_UNSUPPORTED, "ltv_fir: tiled kernel needs block size multiple of 256 (got %d); use b2d_ltv_fir_generic", P);
    if (B > 65535) return fail(B2D_ERR_UNSUPPORTED, "ltv_fir: batch %d > 65535", B);
    const int njobs = ir2 ? 2 : 1;
    {
        const int sel = g_fir_impl.load(std::memory_order_relaxed);
        const int impl = sel == 0 ? fir_auto_impl() : sel;
        const bool tc_ok = (P == 512) && !(njobs == 2 && (taps1 != taps2 || addend));
        if (impl == 4 && ltv_fir_fft_supported(P, taps1, taps2, njobs)) {
            const float* ptrs0[] = {x1, x2, y1, y2, addend, mix};
            for (const float* q : ptrs0)
                if (q && !aligned16(q)) return fail(B2D_ERR_ALIGN, "ltv_fir: signal pointers must be 16-byte aligned");
            if ((taps1 & 1) || (njobs == 2 && (taps2 & 1))) return fail(B2D_ERR_SHAPE, "ltv_fir: bad tap count");
            return ltv_fir_fft_launch(x1, ir1, taps1, y1, x2, ir2, taps2, y2, addend, mix, seed, utt_off, B, nF, P, st);
        }
        if (impl == 2 && !tc_ok) return fail(B2D_ERR_UNSUPPORTED, "ltv_fir: tensor-core kernel needs block size 512");
        if (impl == 2) {
            const float* ptrs0[] = {x1, x2, y1, y2, addend, mix};
            for (const float* q : ptrs0)
                if (q && !aligned16(q)) return fail(B2D_ERR_ALIGN, "ltv_fir: signal pointers must be 16-byte aligned");
            if (taps1 <= 0 || (taps1 & 1) || (njobs == 2 && (taps2 <= 0 || (taps2 & 1)))) return fail(B2D_ERR_SHAPE, "ltv_fir: bad tap count");
            return ltv_fir_tc_launch(x1, ir1, taps1, y1, x2, ir2, taps2, y2, addend, mix, seed, utt_off, B, nF, P, st);
        }
    }
    if (njobs == 2) {
        if (taps2 <= 0 || (taps2 & 1)) return fail(B2D_ERR_SHAPE, "ltv_fir: bad taps2");
        // each job's output tile starts at fP - (L/2+1): only equal tap counts share a tile
        if (taps1 != taps2)
            return fail(B2D_ERR_UNSUPPORTED, "ltv_fir: two jobs must have the same tap count (got %d, %d)", taps1, taps2);
        if (njobs * (P / 8) > 512) return fail(B2D_ERR_UNSUPPORTED, "ltv_fir: block size too large for two jobs");
    }
    const float* ptrs[] = {x1, x2, y1, y2, addend, mix};
    for (const float* q : ptrs)
        if (q && !aligned16(q)) return fail(B2D_ERR_ALIGN, "ltv_fir: signal pointers must be 16-byte aligned");
    FirParams p;
    p.job[0] = {x1, ir1, y1, taps1};
    p.job[1] = {x2, ir2, y2, njobs == 2 ? taps2 : taps1};
    p.njobs = njobs;
    p.addend = addend;
    p.mix = mix;
    p.seed = seed;
    p.utt_off = utt_off;
    p.nF = nF; p.P = P; p.T = nF * P;
    const int Mh = taps1 / 2 + 1;
    const int ntiles = nF + (Mh + P - 1) / P;
    const size_t smem = (size_t)(njobs * (6 * P + 8) + njobs * P) * sizeof(float);
    const int threads = njobs * (P / 8);
    auto go = [&](auto kern) -> int {
        if (smem > 48 * 1024) {
            cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) return fail((int)e, "ltv_fir: smem attr: %s", cudaGetErrorString(e));
        }
        cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        kern<<<dim3(ntiles, B), threads, smem, st>>>(p);
        return check_launch("ltv_fir");
    };
    if (g_fir_variant.load(std::memory_order_relaxed) != 1 && P % 512 == 0) {            // 16 outputs/thread, register pairs (one warp per filter at P = 512)
        const int threads16 = njobs * (P / 16);
        const size_t smem = (size_t)(njobs * (6 * P + 8 + P + (P >> 4) + 8) + P) * sizeof(float);
        auto go16 = [&](auto kern) -> int {
            if (smem > 48 * 1024) {
                cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
                if (e != cudaSuccess) return fail((int)e, "ltv_fir16: smem attr: %s", cudaGetErrorString(e));
            }
            cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            kern<<<dim3(ntiles, B), threads16, smem, st>>>(p);
            return check_launch("ltv_fir16");
        };
        if (threads16 <= 64) return go16(ltv_fir16_kernel<64, 7>);
        return go16(ltv_fir16_kernel<256, 1>);
    }
    // register budget: 80/thread is spill-free; more resident CTAs hide the table-build prologue
    if (threads <= 128) return go(ltv_fir_kernel<128, 6>);
    if (threads <= 256) return go(ltv_fir_kernel<256, 3>);
    return go(ltv_fir_kernel<512, 1>);
}

}  // namespace b2d

extern "C" int b2d_set_fir_impl(int impl) {
    // 0 auto, 1 CUDA cores (auto variant), 2 tensor cores, 3 CUDA cores forcing the 8-outputs/thread scalar kernel,
    // 4 FFT domain
    if (impl < 0 || impl > 4) return b2d::fail(B2D_ERR_UNSUPPORTED, "set_fir_impl: %d", impl);
    b2d::g_fir_impl.store((impl == 3) ? 1 : impl, std::memory_order_relaxed);
    b2d::g_fir_variant.store((impl == 3) ? 1 : 0, std::memory_order_relaxed);
    return 0;
}

extern "C" int b2d_ltv_fir(const float* x1, const float* ir1, int taps1, float* y1, const float* x2,
                           const float* ir2, int taps2, float* y2, float* mix, uint64_t seed,
                           int64_t utterance_offset, int B, int n_frames, int block, void* stream) {
    return b2d::ltv_fir_launch(x1, ir1, taps1, y1, x2, ir2, taps2, y2, nullptr, mix, seed, utterance_offset, B,
                               n_frames, block, (cudaStream_t)stream);
}

extern "C" int b2d_ltv_fir_generic(const float* x, const float* ir, int taps, float* y, int B, int n_frames,
                                   int block, void* stream) {
    if (!x || !ir || !y) return b2d::fail(B2D_ERR_NULL, "ltv_fir_generic: null pointer");
    if (B <= 0 || n_frames <= 0 || block <= 0 || taps <= 0) return b2d::fail(B2D_ERR_SHAPE, "ltv_fir_generic: bad shape");
    if (B > 65535) return b2d::fail(B2D_ERR_UNSUPPORTED, "ltv_fir_generic: batch %d > 65535", B);
    const int T = n_frames * block;
    ltv_fir_generic_kernel<<<dim3((T + 255) / 256, B), 256, 0, (cudaStream_t)stream>>>(x, ir, taps, y, n_frames, block, T);
    return b2d::check_launch("ltv_fir_generic");
}
