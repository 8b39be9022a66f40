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
//     (TMA) on an mbarrier, double buffered, one chunk ahead;
//   * per chunk of 16 bins all threads evaluate pi*tanh(c) (coalesced), 64 threads carry the
//     per-frame running sum (sequential along K: fp64 accumulate / fp32 emit like torch's CPU
//     cumsum), then all threads evaluate sincos / exp, split into tf32 hi + lo and write the A
//     operand chunk to shared memory;
//   * warpgroup w owns the 16-column tiles w, w + 4, ... of every accumulator (Ce | Se | Co | So), in
//     registers: it loads its A fragments from shared memory into registers and issues 3 wgmmas
//     (hi*hi, lo*hi, hi*lo) per accumulator tile, B straight from the TMA-filled stage;
//   * epilogue: each thread holds all accumulators of its (frame, column) pairs, forms the four taps per
//     column, applies the window and stores them.
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
constexpr int kABlock = kRows * 8;       // floats per A block: [64 rows][4 k pairs (k, k + 4)]
constexpr int kAccRegs = 64;             // accumulator registers per thread: NACC x (16-column tiles per warpgroup) x 8

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
// D[64 x 16] += A[64 x 8] (registers, tf32) . B[8 x 16] (shared memory, tf32)
__device__ __forceinline__ void wgmma_tf32_m64n16k8(float (&d)[8], const uint32_t (&a)[4], uint64_t db) {
    asm volatile("wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, 1, 1, 1;\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db));
}
// keeps a register live (and unmoved) across asynchronous wgmma reads of it
__device__ __forceinline__ void fence_reg(float& r) { asm volatile("" : "+f"(r)::"memory"); }
__device__ __forceinline__ void fence_reg(uint32_t& r) { asm volatile("" : "+r"(r)::"memory"); }

struct IrTcParams {
    const float* c;
    long long ctrl_stride;
    const float* f0;
    const float* image;      // tensor-core table image
    int n_total, M;
    float hw_num;
    float* ir;
};

// MODE as in b200ddsp.h.  NACC = 4 (all-pass: Ce Se Co So; Npad <= 128) or 2 (magnitude: Ce Co; Npad <= 256): either
// way NACC x JT tiles x 8 = 64 accumulator registers per thread.  ROWS = frames a CTA actually fills of its 64 tile
// rows: 64, or 32 for small launches (latency bound: the activations and the write-out scale with the rows, the MMAs do
// not care -- a D row depends on its own A row only; the unused A rows are never written and their D rows never read).
template <int MODE, int ROWS>
__global__ void __launch_bounds__(kThreads, 1) ir_build_tc_kernel(IrTcParams p) {
    constexpr bool kAllpass = (MODE == B2D_IR_ALLPASS);
    constexpr int NACC = kAllpass ? 4 : 2;
    constexpr int JT = kAccRegs / (8 * NACC);                      // 16-column tiles per warpgroup
    static_assert(ROWS == 32 || ROWS == 64, "rows per CTA");
    constexpr int rows = ROWS, urows = ROWS >> 5;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    const int M = p.M, L = 2 * (M - 1), Nt = (M - 1) / 2 + 1;
    const int Npad = b2d::tc_npad(M), NC = b2d::tc_kpad(M) / 8, NT16 = Npad / 16;
    const int bblock = Npad * 8;                                   // floats per B block
    const int sa_floats = NACC * 2 * kABlock, sb_floats = NACC * 2 * bblock;
    float* sA0 = reinterpret_cast<float*>(smem_raw);               // [2 stages][kind][hi|lo][64 rows][4][2]
    float* sB0 = sA0 + 2 * sa_floats;                              // [2 stages][table][hi|lo][2 k-chunks][Npad][4]
    float* wtab = sB0 + 2 * sb_floats;                             // [L] Hann window (MAG_HANN)
    float* gds = wtab + ((L + 3) & ~3);                            // [64][17] pi*tanh(c) of the chunk, then the fp32 phase
    __shared__ __align__(8) uint64_t b_full[2];

    const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127, lane = tid & 31;
    const int F0 = blockIdx.x * rows;
    const float invL = 1.0f / (float)L;

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
    }
    if (MODE == B2D_IR_MAG_HANN)
        for (int i = tid; i < L; i += kThreads) wtab[i] = 0.5f - 0.5f * cospif(2.0f * invL * (float)i);
    __syncthreads();

    float acc[NACC][JT][8];
#pragma unroll
    for (int a = 0; a < NACC; ++a)
#pragma unroll
        for (int j = 0; j < JT; ++j)
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[a][j][i] = 0.f;

    double run = 0.0;      // threads 0..rows-1: group-delay cumsum of frame F0 + tid (fp64 accumulate, fp32 emit)

    // raw controls of a chunk (element e = tid + 512 u -> row e >> 4, bin 16 ch + (e & 15)); fetched one chunk ahead so
    // the global-load latency hides behind the previous chunk's barriers
    float cpre[urows];
    auto fetch = [&](int ch) {
#pragma unroll
        for (int u = 0; u < urows; ++u) {
            const int e = tid + u * kThreads, row = e >> 4, m = 16 * ch + (e & 15);
            cpre[u] = (m < M && F0 + row < p.n_total) ? __ldg(p.c + (size_t)(F0 + row) * p.ctrl_stride + m) : 0.f;
        }
    };
    fetch(0);

    for (int ch = 0; ch < NC; ++ch) {
        const int st = ch & 1;
        float* sA = sA0 + st * sa_floats;                          // A blocks: [kind][hi|lo][64][4][2]
        const float* sB = sB0 + st * sb_floats;
        // element e = (row, i): bins 16 ch + i, i = 0..15;  16 lanes per row
        if (kAllpass) {
            // phase 1: pi * tanh(c)   (:581)
#pragma unroll
            for (int u = 0; u < urows; ++u) {
                const int e = tid + u * kThreads, row = e >> 4, i = e & 15, m = 16 * ch + i;
                float g = 0.f;
                if (m < M && F0 + row < p.n_total) g = B2D_PI_F * tanhf(cpre[u]);
                gds[row * 17 + i] = g;
            }
            if (ch + 1 < NC) fetch(ch + 1);
            __syncthreads();
            // phase 2: running sum per frame, fp64 accumulate / fp32 emit   (:599, torch CPU cumsum)
            if (tid < rows) {
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    run += (double)gds[tid * 17 + i];
                    gds[tid * 17 + i] = (float)run;
                }
            }
            __syncthreads();
        }
        // phase 3: spectrum values -> tf32 hi/lo -> A operand blocks
#pragma unroll
        for (int u = 0; u < urows; ++u) {
            const int e = tid + u * kThreads, row = e >> 4, i = e & 15, m = 16 * ch + i;
            const bool act = (m < M) && (F0 + row < p.n_total);
            const float wgt = ((m == 0 || m == M - 1) ? 1.0f : 2.0f) * invL;
            float r = 0.f, im = 0.f;
            if (kAllpass) {
                if (act) {
                    const double t = (double)gds[row * 17 + i];
                    const double kk = rint(t * 0.15915494309189535);
                    const float rr = (float)fma(-kk, 6.283185307179586, t);   // exact reduction of the fp32 phase
                    float sn, cs;
                    __sincosf(rr, &sn, &cs);
                    r = cs * wgt; im = sn * wgt;
                }
            } else if (act) {
                float v = expf(cpre[u]);
                if (MODE == B2D_IR_MAG_HANN) v *= 0.0078125f;
                r = v * wgt;
            }
            // A element (row, k) of parity par: k and k + 4 side by side, the pair a thread's fragment needs
            const int par = i & 1, k = i >> 1;
            const int pos = row * 8 + (k & 3) * 2 + (k >> 2);
            float h, l;
            split_tf32(r, h, l);
            const int kindR = kAllpass ? 2 * par : par;            // all-pass kinds: Re, Ie, Ro, Io ; magnitude: Re, Ro
            sA[(kindR * 2 + 0) * kABlock + pos] = h;
            sA[(kindR * 2 + 1) * kABlock + pos] = l;
            if (kAllpass) {
                split_tf32(im, h, l);
                sA[((2 * par + 1) * 2 + 0) * kABlock + pos] = h;
                sA[((2 * par + 1) * 2 + 1) * kABlock + pos] = l;
            }
        }
        if (!kAllpass && ch + 1 < NC) fetch(ch + 1);
        __syncthreads();
        // the other stage's last readers (chunk ch - 1's wgmmas) completed before this barrier: prefetch into it
        if (tid == 0 && ch + 1 < NC) load_tables(ch + 1);

        // ---- MMAs of warpgroup wg: A fragments (rows 16 warp + lane / 4 (+ 8), k = lane % 4 (+ 4)) from shared memory ----
        uint32_t af[NACC][2][4];
        {
            const int r0 = 16 * (wtid >> 5) + (lane >> 2), kq = lane & 3;
#pragma unroll
            for (int a = 0; a < NACC; ++a)
#pragma unroll
                for (int hl = 0; hl < 2; ++hl) {
                    const float* blk = sA + (a * 2 + hl) * kABlock;
                    const float2 v0 = *reinterpret_cast<const float2*>(blk + r0 * 8 + kq * 2);
                    const float2 v1 = *reinterpret_cast<const float2*>(blk + (r0 + 8) * 8 + kq * 2);
                    af[a][hl][0] = __float_as_uint(v0.x); af[a][hl][1] = __float_as_uint(v1.x);
                    af[a][hl][2] = __float_as_uint(v0.y); af[a][hl][3] = __float_as_uint(v1.y);
                }
        }
        b2d::mbar_wait(&b_full[st], (uint32_t)((ch >> 1) & 1));
#pragma unroll
        for (int a = 0; a < NACC; ++a)
#pragma unroll
            for (int j = 0; j < JT; ++j)
#pragma unroll
                for (int i = 0; i < 8; ++i) fence_reg(acc[a][j][i]);
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
        {
            const uint32_t b0 = b2d::smem_u32(sB);
            const uint32_t lbo_b = (uint32_t)Npad * 16;
#pragma unroll
            for (int j = 0; j < JT; ++j) {
                // 16-column tile: columns 16 t .. 16 t + 15.  A tile past Npad recomputes the last one (never stored):
                // a branch around wgmma would make ptxas serialise every wgmma of the kernel
                const int t = min(wg + 4 * j, NT16 - 1);
#pragma unroll
                for (int a = 0; a < NACC; ++a) {
                    // accumulator a pairs A kind a with table a (all-pass: Re.cosE, Ie.sinE, Ro.cosO, Io.sinO)
                    const uint32_t bh = b0 + (uint32_t)((a * 2 + 0) * bblock * 4 + t * 256);
                    const uint32_t bl = b0 + (uint32_t)((a * 2 + 1) * bblock * 4 + t * 256);
                    wgmma_tf32_m64n16k8(acc[a][j], af[a][0], make_desc(bh, lbo_b, 128));
                    wgmma_tf32_m64n16k8(acc[a][j], af[a][1], make_desc(bh, lbo_b, 128));
                    wgmma_tf32_m64n16k8(acc[a][j], af[a][0], make_desc(bl, lbo_b, 128));
                }
            }
        }
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
        for (int a = 0; a < NACC; ++a) {
#pragma unroll
            for (int hl = 0; hl < 2; ++hl)
#pragma unroll
                for (int i = 0; i < 4; ++i) fence_reg(af[a][hl][i]);
#pragma unroll
            for (int j = 0; j < JT; ++j)
#pragma unroll
                for (int i = 0; i < 8; ++i) fence_reg(acc[a][j][i]);
        }
    }

    // ---- epilogue: accumulator register i of tile j holds row 16 warp + lane / 4 + 8 ((i >> 1) & 1),
    //      column 16 t + 8 (i >> 2) + 2 (lane % 4) + (i & 1) ----
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
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
        const int row = 16 * (wtid >> 5) + (lane >> 2) + 8 * hrow;
        if (row >= rows || F0 + row >= p.n_total) continue;
        float hw = 1.f;
        if (MODE == B2D_IR_MAG_DYNAMIC) hw = p.hw_num / (p.f0[F0 + row] + 1e-3f);
        float* dst = p.ir + (size_t)(F0 + row) * L;
#pragma unroll
        for (int j = 0; j < JT; ++j) {
            const int t = wg + 4 * j;
            if (t >= NT16) continue;
#pragma unroll
            for (int s = 0; s < 2; ++s)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int i = 4 * s + 2 * hrow + e;
                    const int tl = 16 * t + 8 * s + 2 * (lane & 3) + e, th = M - 1 - tl;
                    if (tl >= Nt) continue;
                    const float Ce = acc[0][j][i], Co = acc[kAllpass ? 2 : 1][j][i];
                    const float Se = kAllpass ? acc[1][j][i] : 0.f, So = kAllpass ? acc[3][j][i] : 0.f;
                    const float Cl = Ce + Co, Ch = Ce - Co;
                    const float Sl = Se + So, Sh = So - Se;
                    // taps: M-1+tl, M-1-tl, M-1+th, M-1-th = tl
                    if (tl <= M - 2) dst[M - 1 + tl] = (Cl - Sl) * window(M - 1 + tl, hw);
                    if (tl >= 1) dst[M - 1 - tl] = (Cl + Sl) * window(M - 1 - tl, hw);
                    if (th != tl && th <= M - 2) dst[M - 1 + th] = (Ch - Sh) * window(M - 1 + th, hw);
                    if (th != tl && th >= 1) dst[tl] = (Ch + Sh) * window(tl, hw);
                }
        }
    }
}

size_t tc_smem_bytes(int nacc, int M) {
    const int Npad = b2d::tc_npad(M), L = 2 * (M - 1);
    return (size_t)2 * (nacc * 2 * kABlock + nacc * 2 * Npad * 8) * 4 + (size_t)((L + 3) & ~3) * 4 + (size_t)kRows * 17 * 4;
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
