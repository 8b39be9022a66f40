// K3-TC: impulse responses from raw controls on the Hopper tensor cores (wgmma tf32, 3xTF32).
// Same math as ir_build.cu (reference ddsp/core.py:254-270 + windows + activations): per frame
//   C(t) = Ce + Co, C(M-1-t) = Ce - Co, S(t) = Se + So, S(M-1-t) = So - Se,
//   Ce[t] = sum_{m even} R_m cos(w m t), Se = sum_{m even} I_m sin(w m t), (Co, So: odd m)
// i.e. four GEMMs  [frames x K] . [K x Nt]  against CONSTANT tables -- a proper GEMM (M = 64 frames
// per CTA, N = Nt <= 128 columns, K = 128 bins per parity), unlike the FIR: every table element is
// reused by 64 frames, so the operands are worth their shared-memory traffic.
//
// Pipeline per CTA (64 frames = one wgmma M tile, 512 threads = 4 warpgroups):
//   * tables live in global memory already in the K-major no-swizzle operand image, hi/lo split,
//     one contiguous block per (chunk of 8 K, table): they are fetched with 1-D bulk async copies
//     (TMA) on an mbarrier, double buffered, two chunks ahead;
//   * software pipeline over chunks of 16 bins, one block barrier per chunk: every warpgroup issues the
//     asynchronous wgmmas of chunk c, then, while they run, all threads evaluate pi*tanh(c) of chunk
//     c + 3 (coalesced), 64 threads carry the per-frame running sum of chunk c + 2 (sequential along K:
//     fp64 accumulate / fp32 emit like torch's CPU cumsum) and all threads evaluate sincos of chunk
//     c + 1 (magnitude: exp of chunk c + 1), split into tf32 hi + lo and write it to the other A stage;
//   * warpgroup w owns a contiguous block of columns of every accumulator (Ce | Se | Co | So), in
//     registers, and issues 3 wgmmas (hi*hi, lo*hi, hi*lo) per accumulator, A and B both read from
//     shared memory through K-major no-swizzle descriptors;
//   * epilogue: each thread holds all accumulators of its (frame, column) pairs, forms the four taps per
//     column and applies the window into shared memory; the CTA stores them in contiguous 16-byte runs.
// fp32 tensor-core accumulation truncates (~0.5 ulp per step, 48 steps per accumulator): <= 3e-6 relative
// gain error on the taps, far below the parity gate.
#include "b2d_common.cuh"

namespace b2d {
// layout helpers shared with b2d_dft_tables (ir_build.cu)
__host__ __device__ inline int tc_npad(int M) { return (((M - 1) / 2 + 1) + 15) & ~15; }
__host__ __device__ inline int tc_kpad(int M) { return (((M + 1) / 2) + 7) & ~7; }
__host__ __device__ inline size_t tc_block_floats(int M) { return (size_t)tc_npad(M) * 8; }   // one (chunk, table, hi|lo) block
__host__ __device__ inline size_t tc_image_floats(int M) { return (size_t)(tc_kpad(M) / 8) * 8 * tc_block_floats(M); }
}  // namespace b2d

namespace {

constexpr int kThreads = 512;
constexpr int kRows = 64;                // frames per CTA = wgmma M
constexpr int kABlock = kRows * 8;       // floats per A block: [2 k-chunks][64 rows][4]
constexpr int kAccRegs = 64;             // accumulator registers per thread: NACC x (columns per warpgroup) / 2

__device__ __forceinline__ uint32_t tf32_rn_bits(float x) {
    uint32_t u = __float_as_uint(x);
    u += 0x00000FFFu + ((u >> 13) & 1u);
    return u & 0xFFFFE000u;
}
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    hi = __uint_as_float(tf32_rn_bits(x));
    lo = __uint_as_float(tf32_rn_bits(x - hi));
}
// wgmma shared-memory descriptor, K-major, no swizzle: LBO = byte stride between the two core matrices along K,
// SBO = byte stride between 8-row groups
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFF);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
    return d;
}
// D[64 x N] += A[64 x 8] . B[8 x N], both tf32 from shared memory (descriptors)
__device__ __forceinline__ void wgmma_tf32_k8(float (&d)[16], uint64_t da, uint64_t db) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, 1, 1, 1;\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(da), "l"(db));
}
__device__ __forceinline__ void wgmma_tf32_k8(float (&d)[32], uint64_t da, uint64_t db) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, 1, 1, 1;\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(da), "l"(db));
}
// keeps an accumulator register unmoved across the asynchronous wgmma writes of it
__device__ __forceinline__ void fence_reg(float& r) { asm volatile("" : "+f"(r)::"memory"); }

struct IrTcParams {
    const float* c;
    long long ctrl_stride;
    const float* f0;
    const float* image;      // tensor-core table image
    int n_total, M;
    float hw_num;
    float* ir;
};

// MODE as in b200ddsp.h.  NACC = 4 (all-pass: Ce Se Co So; Npad <= 128) or 2 (magnitude: Ce Co; Npad <= 256).
// Warpgroup w owns the TN columns [TN w, TN w + TN) of every accumulator: TN = 32 (all-pass) or 64 (magnitude), either
// way NACC x TN / 2 = 64 accumulator registers per thread.  A warpgroup whose columns all lie past Npad recomputes the
// last tile and stores nothing: a branch around wgmma would make ptxas serialise every wgmma of the kernel.
// ROWS = frames a CTA actually fills of its 64 tile rows: 64, or 32 for small launches (latency bound: the activations
// and the write-out scale with the rows, the MMAs do not care -- a D row depends on its own A row only; the unused A rows
// are never written and their D rows never read).
// 96 registers: 512 x 96 leaves a quarter of the register file, room for one 128-thread oscillator-bank CTA (128 registers
// per thread) on the same SM while the bank runs beside the impulse-response builds.
template <int MODE, int ROWS>
__global__ void __maxnreg__(96) ir_build_tc_kernel(IrTcParams p) {
    constexpr bool kAllpass = (MODE == B2D_IR_ALLPASS);
    constexpr int NACC = kAllpass ? 4 : 2;
    constexpr int TN = kAccRegs * 2 / NACC;                        // columns per warpgroup
    constexpr int NREG = TN / 2;                                   // accumulator registers per thread and accumulator
    // software-pipeline depth: step s of the activations consumes the controls of chunk s; the MMAs of chunk c are issued
    // at step c + LAG.  All-pass: step s evaluates pi*tanh of chunk s, scans chunk s - 1, writes the A operand of chunk
    // s - 2.  Magnitude: step s writes the A operand of chunk s.
    constexpr int LAG = kAllpass ? 3 : 1;
    static_assert(ROWS == 32 || ROWS == 64, "rows per CTA");
    constexpr int rows = ROWS, urows = ROWS >> 5;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int M = p.M, L = 2 * (M - 1), Nt = (M - 1) / 2 + 1;
    const int Npad = b2d::tc_npad(M), NC = b2d::tc_kpad(M) / 8;
    const int bblock = Npad * 8;                                   // floats per B block
    const int sa_floats = NACC * 2 * kABlock, sb_floats = NACC * 2 * bblock;
    float* sA0 = reinterpret_cast<float*>(smem_raw);               // [2 stages][kind][hi|lo][2 k-chunks][64 rows][4]
    float* sB0 = sA0 + 2 * sa_floats;                              // [2 stages][table][hi|lo][2 k-chunks][Npad][4]
    float* stage_out = sA0;                                        // epilogue, over the operand stages: [32][L] taps
    // TN * 4 floats of slack for the B columns a last partial tile reads past Npad
    float* wtab = sA0 + max(2 * sa_floats + 2 * sb_floats + TN * 4, 32 * L);   // [L] Hann window (MAG_HANN)
    float* gds = wtab + ((L + 3) & ~3);                            // all-pass: [4 slots][64][17] pi*tanh(c), then phase
    __shared__ __align__(8) uint64_t b_full[2];

    const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127, lane = tid & 31;
    const int F0 = blockIdx.x * rows;
    const float invL = 1.0f / (float)L;
    const int col0 = min(wg, (Npad - 1) / TN) * TN;                // first column of this warpgroup's MMAs

    // tables of chunk ch -> stage ch & 1 (TMA bulk copies).  Image: [chunk][cosE hi lo, sinE hi lo, cosO hi lo, sinO hi lo]
    auto load_tables = [&](int ch) {
        float* sB = sB0 + (ch & 1) * sb_floats;
        uint64_t* bar = &b_full[ch & 1];
        b2d::mbar_arrive_expect_tx(bar, (uint32_t)(NACC * 2 * bblock * 4));
        const float* src = p.image + (size_t)ch * 8 * bblock;
        if (kAllpass) {
            b2d::tma_load_1d(sB, src, (uint32_t)(8 * bblock * 4), bar);
        } else {                                                   // cosE hi/lo and cosO hi/lo only
            b2d::tma_load_1d(sB, src, (uint32_t)(2 * bblock * 4), bar);
            b2d::tma_load_1d(sB + 2 * bblock, src + 4 * bblock, (uint32_t)(2 * bblock * 4), bar);
        }
    };
    if (tid == 0) {
        b2d::mbar_init(&b_full[0], 1); b2d::mbar_init(&b_full[1], 1);
        b2d::fence_mbar_init();
        load_tables(0);
        if (NC > 1) load_tables(1);
    }
    if (MODE == B2D_IR_MAG_HANN)
        for (int i = tid; i < L; i += kThreads) wtab[i] = 0.5f - 0.5f * cospif(2.0f * invL * (float)i);

    float acc[NACC][NREG];
#pragma unroll
    for (int a = 0; a < NACC; ++a)
#pragma unroll
        for (int i = 0; i < NREG; ++i) acc[a][i] = 0.f;

    double run = 0.0;      // threads 0..rows-1: group-delay cumsum of frame F0 + tid (fp64 accumulate, fp32 emit)

    // raw controls of a chunk (element e = tid + 512 u -> row e >> 4, bin 16 ch + (e & 15)); fetched one step ahead so
    // the global-load latency hides behind the previous step
    float cpre[urows];
    auto fetch = [&](int ch) {
#pragma unroll
        for (int u = 0; u < urows; ++u) {
            const int e = tid + u * kThreads, row = e >> 4, m = 16 * ch + (e & 15);
            cpre[u] = (m < M && F0 + row < p.n_total) ? __ldg(p.c + (size_t)(F0 + row) * p.ctrl_stride + m) : 0.f;
        }
    };
    // spectrum value (row, bin 16 ch + i) -> tf32 hi/lo -> A operand of chunk ch (K-major, no swizzle: element (row, k) of
    // a block at [k / 4][row][k % 4]; parity par = i & 1 goes to kind par (magnitude: Re) or 2 par, 2 par + 1 (all-pass:
    // Re, Im), k = i >> 1)
    auto put_a = [&](int ch, int row, int i, float r, float im) {
        float* sA = sA0 + (ch & 1) * sa_floats;
        const int par = i & 1, k = i >> 1;
        const int pos = (k >> 2) * (kRows * 4) + row * 4 + (k & 3);
        float h, l;
        split_tf32(r, h, l);
        const int kindR = kAllpass ? 2 * par : par;                // all-pass kinds: Re, Ie, Ro, Io ; magnitude: Re, Ro
        sA[(kindR * 2 + 0) * kABlock + pos] = h;
        sA[(kindR * 2 + 1) * kABlock + pos] = l;
        if (kAllpass) {
            split_tf32(im, h, l);
            sA[((2 * par + 1) * 2 + 0) * kABlock + pos] = h;
            sA[((2 * par + 1) * 2 + 1) * kABlock + pos] = l;
        }
    };
    // one pipeline step (element e = (row, i): bins 16 ch + i, i = 0..15; 16 lanes per row).  The gds slots and the A
    // stage a step writes were last read no later than the previous step, whose MMAs complete before its closing barrier
    auto step = [&](int s) {
        if (kAllpass) {
            if (s < NC) {                                          // pi * tanh(c)   (:581)
                float* g = gds + (s & 3) * (kRows * 17);
#pragma unroll
                for (int u = 0; u < urows; ++u) {
                    const int e = tid + u * kThreads, row = e >> 4, i = e & 15, m = 16 * s + i;
                    float v = 0.f;
                    if (m < M && F0 + row < p.n_total) v = B2D_PI_F * tanhf(cpre[u]);
                    g[row * 17 + i] = v;
                }
                if (s + 1 < NC) fetch(s + 1);
            }
            // running sum per frame, fp64 accumulate / fp32 emit (:599, torch CPU cumsum), sequential along the bins
            if (s >= 1 && s - 1 < NC && tid < rows) {
                float* g = gds + ((s - 1) & 3) * (kRows * 17) + tid * 17;
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    run += (double)g[i];
                    g[i] = (float)run;
                }
            }
            const int ch = s - 2;
            if (ch >= 0 && ch < NC) {
                const float* g = gds + (ch & 3) * (kRows * 17);
#pragma unroll
                for (int u = 0; u < urows; ++u) {
                    const int e = tid + u * kThreads, row = e >> 4, i = e & 15, m = 16 * ch + i;
                    const float wgt = ((m == 0 || m == M - 1) ? 1.0f : 2.0f) * invL;
                    float r = 0.f, im = 0.f;
                    if (m < M && F0 + row < p.n_total) {
                        const double t = (double)g[row * 17 + i];
                        const double kk = rint(t * 0.15915494309189535);
                        const float rr = (float)fma(-kk, 6.283185307179586, t);   // exact reduction of the fp32 phase
                        float sn, cs;
                        __sincosf(rr, &sn, &cs);
                        r = cs * wgt; im = sn * wgt;
                    }
                    put_a(ch, row, i, r, im);
                }
                b2d::fence_proxy_async();                          // generic-proxy writes -> wgmma operand reads
            }
        } else if (s < NC) {
#pragma unroll
            for (int u = 0; u < urows; ++u) {
                const int e = tid + u * kThreads, row = e >> 4, i = e & 15, m = 16 * s + i;
                const float wgt = ((m == 0 || m == M - 1) ? 1.0f : 2.0f) * invL;
                float r = 0.f;
                if (m < M && F0 + row < p.n_total) {
                    float v = expf(cpre[u]);
                    if (MODE == B2D_IR_MAG_HANN) v *= 0.0078125f;
                    r = v * wgt;
                }
                put_a(s, row, i, r, 0.f);
            }
            if (s + 1 < NC) fetch(s + 1);
            b2d::fence_proxy_async();
        }
    };

    fetch(0);
    for (int s = 0; s < LAG; ++s) {
        step(s);
        __syncthreads();
    }
    const uint32_t lbo_a = kRows * 16, lbo_b = (uint32_t)Npad * 16;
    for (int ch = 0; ch < NC; ++ch) {
        const int st = ch & 1;
        // ---- MMAs of chunk ch, in flight while this thread evaluates the activations of the next chunks ----
        b2d::mbar_wait(&b_full[st], (uint32_t)((ch >> 1) & 1));
#pragma unroll
        for (int a = 0; a < NACC; ++a)
#pragma unroll
            for (int i = 0; i < NREG; ++i) fence_reg(acc[a][i]);
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
        {
            const uint32_t a0 = b2d::smem_u32(sA0 + st * sa_floats);
            const uint32_t b0 = b2d::smem_u32(sB0 + st * sb_floats) + (uint32_t)(col0 * 16);
#pragma unroll
            for (int a = 0; a < NACC; ++a) {
                // accumulator a pairs A kind a with table a (all-pass: Re.cosE, Ie.sinE, Ro.cosO, Io.sinO)
                const uint64_t ah = make_desc(a0 + (uint32_t)((a * 2 + 0) * kABlock * 4), lbo_a, 128);
                const uint64_t al = make_desc(a0 + (uint32_t)((a * 2 + 1) * kABlock * 4), lbo_a, 128);
                const uint64_t bh = make_desc(b0 + (uint32_t)((a * 2 + 0) * bblock * 4), lbo_b, 128);
                const uint64_t bl = make_desc(b0 + (uint32_t)((a * 2 + 1) * bblock * 4), lbo_b, 128);
                wgmma_tf32_k8(acc[a], ah, bh);
                wgmma_tf32_k8(acc[a], al, bh);
                wgmma_tf32_k8(acc[a], ah, bl);
            }
        }
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        step(ch + LAG);
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
        for (int a = 0; a < NACC; ++a)
#pragma unroll
            for (int i = 0; i < NREG; ++i) fence_reg(acc[a][i]);
        // publishes the A operand of the next chunk; every warpgroup's MMAs of chunk ch have completed before it
        __syncthreads();
        if (tid == 0 && ch + 2 < NC) load_tables(ch + 2);
    }

    // ---- epilogue: accumulator register i holds row 16 warp + lane / 4 + 8 ((i >> 1) & 1),
    //      column TN wg + 8 (i >> 2) + 2 (lane % 4) + (i & 1).  The taps go out through shared memory (the operand
    //      stages, free now) in two passes, one per half of each warp's rows: every warp forms its taps, then the CTA
    //      stores the four runs of 8 consecutive frames (8 L contiguous floats each) with 16-byte stores instead of
    //      scattering 4-byte ones ----
    auto window = [&](int idx, float hw) -> float {
        if (MODE == B2D_IR_MAG_HANN) return wtab[idx];
        if (MODE == B2D_IR_MAG_DYNAMIC) {                          // (ddsp/core.py:244-246), cos(pi u) via exact reduction
            float u = (float)(idx - (M - 1)) / hw;
            if (u > 1.f) u = 0.f;
            const float r = fmaf(-2.0f, rintf(0.5f * u), u);
            return (1.f + __cosf(B2D_PI_F * r)) * 0.5f;
        }
        return 1.f;
    };
    const bool vec = (reinterpret_cast<uintptr_t>(p.ir) & 15u) == 0;   // runs of 8 L floats keep 16-byte alignment
    const int wr = wtid >> 5;
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
        const int row = 16 * wr + (lane >> 2) + 8 * hrow;
        if (wg * TN < Npad && row < rows && F0 + row < p.n_total) {
            float hw = 1.f;
            if (MODE == B2D_IR_MAG_DYNAMIC) hw = p.hw_num / (p.f0[F0 + row] + 1e-3f);
            float* dst = stage_out + (wr * 8 + (lane >> 2)) * L;   // [4 runs][8 frames][L]
#pragma unroll
            for (int q = 0; q < TN / 8; ++q)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int i = 4 * q + 2 * hrow + e;
                    const int tl = TN * wg + 8 * q + 2 * (lane & 3) + e, th = M - 1 - tl;
                    if (tl >= Nt) continue;
                    const float Ce = acc[0][i], Co = acc[kAllpass ? 2 : 1][i];
                    const float Se = kAllpass ? acc[1][i] : 0.f, So = kAllpass ? acc[3][i] : 0.f;
                    const float Cl = Ce + Co, Ch = Ce - Co;
                    const float Sl = Se + So, Sh = So - Se;
                    // taps: M-1+tl, M-1-tl, M-1+th, M-1-th = tl
                    if (tl <= M - 2) dst[M - 1 + tl] = (Cl - Sl) * window(M - 1 + tl, hw);
                    if (tl >= 1) dst[M - 1 - tl] = (Cl + Sl) * window(M - 1 - tl, hw);
                    if (th != tl && th <= M - 2) dst[M - 1 + th] = (Ch - Sh) * window(M - 1 + th, hw);
                    if (th != tl && th >= 1) dst[tl] = (Ch + Sh) * window(tl, hw);
                }
        }
        __syncthreads();
        // run j: frames F0 + 16 j + 8 hrow ..; a run holds 8 L floats, a multiple of 4, so no float4 straddles two runs
        const int run_len = 8 * L;
        for (int v = 4 * tid; v < (rows / 16) * run_len; v += 4 * kThreads) {
            const int j = v / run_len, o = v - j * run_len;
            const int f = F0 + 16 * j + 8 * hrow;
            const int n = min(8, p.n_total - f) * L;               // valid floats of the run
            float* out = p.ir + (size_t)f * L + o;
            const float* src = stage_out + v;
            if (vec && o + 4 <= n) {
                b2d::st_global_v4(out, *reinterpret_cast<const float4*>(src));
            } else {
                for (int k = 0; k < 4 && o + k < n; ++k) out[k] = src[k];
            }
        }
        __syncthreads();
    }
}

size_t tc_smem_bytes(int nacc, int M) {
    const int Npad = b2d::tc_npad(M), L = 2 * (M - 1), TN = kAccRegs * 2 / nacc;
    const int stages = 2 * (nacc * 2 * kABlock + nacc * 2 * Npad * 8) + TN * 4, front = stages > 32 * L ? stages : 32 * L;
    return (size_t)front * 4 + (size_t)((L + 3) & ~3) * 4 + (nacc == 4 ? (size_t)4 * kRows * 17 * 4 : 0);
}

// table image: [chunk][cosE hi, cosE lo, sinE hi, sinE lo, cosO hi, cosO lo, sinO hi, sinO lo][2 k-chunks][Npad][4]
__global__ void dft_image_kernel(int M, float* __restrict__ img) {
    const int L = 2 * (M - 1), Nt = (M - 1) / 2 + 1, Ke = (M + 1) / 2, Ko = M / 2;
    const int Npad = b2d::tc_npad(M), NC = b2d::tc_kpad(M) / 8;
    const size_t bblock = (size_t)Npad * 8, total = (size_t)NC * 8 * bblock;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        const int ch = (int)(i / (8 * bblock));
        const int rem = (int)(i - (size_t)ch * 8 * bblock);
        const int blk = rem / (int)bblock, in = rem - blk * (int)bblock;
        const int cc = in / (Npad * 4), n = (in - cc * Npad * 4) >> 2, e = in & 3;
        const int k = 8 * ch + 4 * cc + e;
        const int tab = blk >> 1, lo = blk & 1;          // tab: 0 cosE 1 sinE 2 cosO 3 sinO
        const bool odd = tab >= 2, is_sin = tab & 1;
        float v = 0.f;
        if (n < Nt && k < (odd ? Ko : Ke)) {
            const int m = 2 * k + (odd ? 1 : 0);
            const long long idx = ((long long)m * n) % L;
            const double ang = 2.0 * (double)idx / (double)L;
            v = (float)(is_sin ? sinpi(ang) : cospi(ang));
        }
        float h, l;
        split_tf32(v, h, l);
        img[i] = lo ? l : h;
    }
}

template <int MODE>
int launch_tc(const IrTcParams& p, int rows, cudaStream_t st) {
    constexpr int NACC = (MODE == B2D_IR_ALLPASS) ? 4 : 2;
    const size_t smem = tc_smem_bytes(NACC, p.M);
    auto kern = rows == 32 ? ir_build_tc_kernel<MODE, 32> : ir_build_tc_kernel<MODE, 64>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return b2d::fail((int)e, "ir_build_tc: smem attr (%zu B): %s", smem, cudaGetErrorString(e));
    kern<<<(p.n_total + rows - 1) / rows, kThreads, smem, st>>>(p);
    return b2d::check_launch("ir_build_tc");
}

}  // namespace

namespace b2d {

size_t tc_image_floats_host(int M) { return tc_image_floats(M); }

int dft_image_launch(int M, float* img, cudaStream_t st) {
    dft_image_kernel<<<num_sms() * 4, 256, 0, st>>>(M, img);
    return check_launch("dft_image");
}

// tensor-core IR build is available when the accumulators fit their 64 registers per thread and the two stages fit
// shared memory (227 KB per block on H100)
bool ir_tc_supported(int mode, int M) {
    const int nacc = (mode == B2D_IR_ALLPASS) ? 4 : 2;
    if (nacc * tc_npad(M) > 512) return false;
    return tc_smem_bytes(nacc, M) <= 227 * 1024;
}

int ir_build_tc_launch(const float* c, int64_t ctrl_stride, int mode, const float* f0, const float* image, int B,
                       int nF, int M, double sr, float* ir, cudaStream_t st) {
    IrTcParams p;
    p.c = c; p.ctrl_stride = ctrl_stride; p.f0 = f0; p.image = image;
    p.n_total = B * nF; p.M = M; p.hw_num = 1.5f * (float)sr; p.ir = ir;
    // 32 frames per CTA when that still runs as a single wave of one CTA per SM; 64 once the grid fills the GPU anyway
    const int rows = (p.n_total + 31) / 32 <= num_sms() ? 32 : 64;
    switch (mode) {
        case B2D_IR_ALLPASS: return launch_tc<B2D_IR_ALLPASS>(p, rows, st);
        case B2D_IR_MAG_HANN: return launch_tc<B2D_IR_MAG_HANN>(p, rows, st);
        default: return launch_tc<B2D_IR_MAG_DYNAMIC>(p, rows, st);
    }
}

}  // namespace b2d
