// K3: frame-wise impulse responses from raw controls.
// Replaces ddsp/core.py:254-270 (frequency_impulse_response = irfft + window + roll) and the
// activations at ddsp/vocoder.py:581-582,599,606,835-836,845,849-851.
//
// For n_mag = M bins the IR has L = 2(M-1) taps.  With H_m = R_m + j I_m, w = 2 pi / L:
//   g(t) = 1/L [ R_0 + (-1)^t R_{M-1} + 2 sum_{m=1}^{M-2} (R_m cos(w m t) - I_m sin(w m t)) ]
//        = C(t) - S(t),   C even in t, S odd in t,   h[tau] = g(tau - (M-1)) * window[tau].
// Only t in [0, M-1] is needed, and because cos(w m (M-1-t)) = (-1)^m cos(w m t) and
// sin(w m (M-1-t)) = -(-1)^m sin(w m t), splitting the sum into even and odd m gives t and
// M-1-t from the same products:  C(t) = Ce+Co, C(M-1-t) = Ce-Co, S(t) = Se+So, S(M-1-t) = So-Se.
// So per frame the work is four [M/2] x [M/2] matrix-vector products against CONSTANT cos/sin
// tables -- i.e. a GEMM over frames with a fixed B matrix (b2d_dft_tables).  Each CTA takes 16
// frames; a thread owns one output column t' and 16 frames x {Ce,Co,Se,So} accumulators, the
// frame-side operand is broadcast from shared memory as float4, the table is streamed
// coalesced through L1/L2.
//
// Numerics kept from the reference: the group-delay cumsum accumulates in fp64 and emits fp32
// (torch CPU cumsum), exp(j phi) is evaluated on the fp32 phase with an accurate sincos
// (phi reaches +-800 rad), Im of the DC and Nyquist bins is ignored (irfft).
#include "b2d_common.cuh"

namespace {

constexpr int kThreads = 128;
constexpr int kFR = 16;  // frames per CTA

__host__ __device__ inline int n_cols(int M) { return (M - 1) / 2 + 1; }
__host__ __device__ inline int n_even(int M) { return (M + 1) / 2; }
__host__ __device__ inline int n_odd(int M) { return M / 2; }

// tables: cosE[Ke][Nt], cosO[Ko][Nt], sinE[Ke][Nt], sinO[Ko][Nt]
__global__ void dft_tables_kernel(int M, float* __restrict__ tab) {
    const int Nt = n_cols(M), Ke = n_even(M), Ko = n_odd(M), L = 2 * (M - 1);
    const int total = 2 * (Ke + Ko) * Nt;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        int row = i / Nt, t = i - row * Nt;
        int m;
        bool is_sin = false;
        if (row < Ke) m = 2 * row;
        else if (row < Ke + Ko) m = 2 * (row - Ke) + 1;
        else if (row < 2 * Ke + Ko) { m = 2 * (row - Ke - Ko); is_sin = true; }
        else { m = 2 * (row - 2 * Ke - Ko) + 1; is_sin = true; }
        const long long idx = ((long long)m * t) % L;           // exact argument reduction
        const double ang = 2.0 * (double)idx / (double)L;       // in units of pi
        tab[i] = (float)(is_sin ? sinpi(ang) : cospi(ang));
    }
}

struct IrParams {
    const float* c;
    long long ctrl_stride;
    const float* f0;
    const float* tab;
    int n_total;  // B * n_frames
    int M;
    float hw_num;  // 1.5 * sr (fp32, as the reference computes it)
    float* ir;
};

template <int MODE>
__global__ void __launch_bounds__(kThreads) ir_build_kernel(IrParams p) {
    constexpr bool kAllpass = (MODE == B2D_IR_ALLPASS);
    extern __shared__ __align__(16) float sm[];
    const int M = p.M, L = 2 * (M - 1), Nt = n_cols(M), Ke = n_even(M), Ko = n_odd(M);
    float* atr = sm;                       // [M][kFR]  weighted Re H, transposed
    float* ati = sm + (size_t)M * kFR;     // [M][kFR]  weighted Im H (all-pass only)
    const int F0 = blockIdx.x * kFR;
    const int nfr = min(kFR, p.n_total - F0);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float invL = 1.0f / (float)L;

    // ---- prologue: activations -> weighted spectra in shared memory ----
    if (kAllpass) {
        // one warp per frame: fp64 inclusive scan of pi*tanh(c) over the bins
        const int per = (M + 31) / 32;
        for (int fr = warp; fr < kFR; fr += kThreads / 32) {
            const bool live = fr < nfr;
            const float* crow = p.c + (size_t)(F0 + (live ? fr : 0)) * p.ctrl_stride;
            const int m0 = lane * per, m1 = min(M, m0 + per);
            double local = 0.0;
            for (int m = m0; m < m1; ++m) local += (double)(B2D_PI_F * tanhf(crow[m]));
            double incl = local;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                double up = __shfl_up_sync(0xffffffffu, incl, d);
                if (lane >= d) incl += up;
            }
            double run = incl - local;
            for (int m = m0; m < m1; ++m) {
                run += (double)(B2D_PI_F * tanhf(crow[m]));
                float s, cth;
                sincosf((float)run, &s, &cth);
                const float wgt = ((m == 0 || m == M - 1) ? 1.0f : 2.0f) * invL;
                atr[m * kFR + fr] = live ? cth * wgt : 0.f;
                ati[m * kFR + fr] = live ? s * wgt : 0.f;
            }
        }
    } else {
        for (int i = tid; i < kFR * M; i += kThreads) {
            const int fr = i / M, m = i - fr * M;
            float v = 0.f;
            if (fr < nfr) {
                const float c = p.c[(size_t)(F0 + fr) * p.ctrl_stride + m];
                v = expf(c);
                if (MODE == B2D_IR_MAG_HANN) v *= 0.0078125f;
                v *= ((m == 0 || m == M - 1) ? 1.0f : 2.0f) * invL;
            }
            atr[m * kFR + fr] = v;
        }
    }
    __syncthreads();

    const float* cosE = p.tab;
    const float* cosO = cosE + (size_t)Ke * Nt;
    const float* sinE = cosO + (size_t)Ko * Nt;
    const float* sinO = sinE + (size_t)Ke * Nt;

    for (int t = tid; t < Nt; t += kThreads) {
        float Ce[kFR], Co[kFR], Se[kFR], So[kFR];
#pragma unroll
        for (int f = 0; f < kFR; ++f) Ce[f] = Co[f] = Se[f] = So[f] = 0.f;

#pragma unroll 2
        for (int k = 0; k < Ke; ++k) {
            const float bc = __ldg(cosE + (size_t)k * Nt + t);
            const float4* ar = reinterpret_cast<const float4*>(atr + (2 * k) * kFR);
#pragma unroll
            for (int q = 0; q < kFR / 4; ++q) {
                const float4 a = ar[q];
                Ce[4 * q + 0] = fmaf(a.x, bc, Ce[4 * q + 0]);
                Ce[4 * q + 1] = fmaf(a.y, bc, Ce[4 * q + 1]);
                Ce[4 * q + 2] = fmaf(a.z, bc, Ce[4 * q + 2]);
                Ce[4 * q + 3] = fmaf(a.w, bc, Ce[4 * q + 3]);
            }
            if (kAllpass) {
                const float bs = __ldg(sinE + (size_t)k * Nt + t);
                const float4* ai = reinterpret_cast<const float4*>(ati + (2 * k) * kFR);
#pragma unroll
                for (int q = 0; q < kFR / 4; ++q) {
                    const float4 a = ai[q];
                    Se[4 * q + 0] = fmaf(a.x, bs, Se[4 * q + 0]);
                    Se[4 * q + 1] = fmaf(a.y, bs, Se[4 * q + 1]);
                    Se[4 * q + 2] = fmaf(a.z, bs, Se[4 * q + 2]);
                    Se[4 * q + 3] = fmaf(a.w, bs, Se[4 * q + 3]);
                }
            }
        }
#pragma unroll 2
        for (int k = 0; k < Ko; ++k) {
            const float bc = __ldg(cosO + (size_t)k * Nt + t);
            const float4* ar = reinterpret_cast<const float4*>(atr + (2 * k + 1) * kFR);
#pragma unroll
            for (int q = 0; q < kFR / 4; ++q) {
                const float4 a = ar[q];
                Co[4 * q + 0] = fmaf(a.x, bc, Co[4 * q + 0]);
                Co[4 * q + 1] = fmaf(a.y, bc, Co[4 * q + 1]);
                Co[4 * q + 2] = fmaf(a.z, bc, Co[4 * q + 2]);
                Co[4 * q + 3] = fmaf(a.w, bc, Co[4 * q + 3]);
            }
            if (kAllpass) {
                const float bs = __ldg(sinO + (size_t)k * Nt + t);
                const float4* ai = reinterpret_cast<const float4*>(ati + (2 * k + 1) * kFR);
#pragma unroll
                for (int q = 0; q < kFR / 4; ++q) {
                    const float4 a = ai[q];
                    So[4 * q + 0] = fmaf(a.x, bs, So[4 * q + 0]);
                    So[4 * q + 1] = fmaf(a.y, bs, So[4 * q + 1]);
                    So[4 * q + 2] = fmaf(a.z, bs, So[4 * q + 2]);
                    So[4 * q + 3] = fmaf(a.w, bs, So[4 * q + 3]);
                }
            }
        }

        // ---- epilogue: t_lo = t, t_hi = M-1-t; h[M-1+u] = C(u)-S(u), h[M-1-u] = C(u)+S(u) ----
        const int tl = t, th = M - 1 - t;
        // tap indices written by this thread
        const int i0 = M - 1 + tl, i1 = M - 1 - tl, i2 = M - 1 + th, i3 = M - 1 - th;
        const bool w0 = tl <= M - 2, w1 = tl >= 1, w2 = (th != tl) && th <= M - 2, w3 = (th != tl) && th >= 1;
        float win0 = 1.f, win1 = 1.f, win2 = 1.f, win3 = 1.f;
        if (MODE == B2D_IR_MAG_HANN) {  // periodic Hann over L taps (ddsp/core.py:211,221)
            const float s = 2.0f * invL;
            win0 = 0.5f - 0.5f * cospif(s * (float)i0);
            win1 = 0.5f - 0.5f * cospif(s * (float)i1);
            win2 = 0.5f - 0.5f * cospif(s * (float)i2);
            win3 = 0.5f - 0.5f * cospif(s * (float)i3);
        }
#pragma unroll
        for (int f = 0; f < kFR; ++f) {
            if (f >= nfr) break;
            float* h = p.ir + (size_t)(F0 + f) * L;
            if (MODE == B2D_IR_MAG_DYNAMIC) {  // per-frame raised cosine (ddsp/core.py:240-251)
                const float hw = p.hw_num / (p.f0[F0 + f] + 1e-3f);
                auto dyn = [&](int idx) {
                    float u = (float)(idx - (M - 1)) / hw;
                    if (u > 1.f) u = 0.f;
                    return (1.f + cosf(B2D_PI_F * u)) * 0.5f;
                };
                win0 = dyn(i0); win1 = dyn(i1); win2 = dyn(i2); win3 = dyn(i3);
            }
            const float Cl = Ce[f] + Co[f], Ch = Ce[f] - Co[f];
            const float Sl = Se[f] + So[f], Sh = So[f] - Se[f];
            if (w0) h[i0] = (Cl - Sl) * win0;
            if (w1) h[i1] = (Cl + Sl) * win1;
            if (w2) h[i2] = (Ch - Sh) * win2;
            if (w3) h[i3] = (Ch + Sh) * win3;
        }
    }
}

template <int MODE>
int launch(const IrParams& p, cudaStream_t st) {
    const size_t smem = (size_t)p.M * kFR * 4 * (MODE == B2D_IR_ALLPASS ? 2 : 1);
    auto kern = ir_build_kernel<MODE>;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return b2d::fail((int)e, "ir_build: smem attr: %s", cudaGetErrorString(e));
    }
    const int grid = (p.n_total + kFR - 1) / kFR;
    kern<<<grid, kThreads, smem, st>>>(p);
    return b2d::check_launch("ir_build");
}

}  // namespace

namespace b2d {
// tensor-core path (ir_build_tc.cu)
int dft_image_launch(int M, float* img, cudaStream_t st);
bool ir_tc_supported(int mode, int M);
int ir_build_tc_launch(const float* c, int64_t ctrl_stride, int mode, const float* f0, const float* image, int B,
                       int nF, int M, double sr, float* ir, cudaStream_t st);
size_t tc_image_floats_host(int M);
// 0 = auto (tensor cores when supported), 1 = CUDA cores, 2 = tensor cores
static std::atomic<int> g_ir_impl{0};   // debug A/B switch, read once per call
static inline size_t cc_table_bytes(int n_mag) {
    const size_t b = (size_t)2 * (n_even(n_mag) + n_odd(n_mag)) * n_cols(n_mag) * sizeof(float);
    return (b + 255) / 256 * 256;
}
}  // namespace b2d

// buffer layout: [CUDA-core tables, padded to 256 B][tensor-core operand image]
extern "C" size_t b2d_dft_tables_bytes(int n_mag) {
    if (n_mag < 2) return 0;
    return b2d::cc_table_bytes(n_mag) + b2d::tc_image_floats_host(n_mag) * sizeof(float);
}

extern "C" int b2d_set_ir_impl(int impl) {
    if (impl < 0 || impl > 2) return b2d::fail(B2D_ERR_UNSUPPORTED, "set_ir_impl: %d", impl);
    b2d::g_ir_impl.store(impl, std::memory_order_relaxed);
    return 0;
}

extern "C" int b2d_dft_tables(int n_mag, float* dft_tables, void* stream) {
    if (!dft_tables) return b2d::fail(B2D_ERR_NULL, "dft_tables: null pointer");
    if (n_mag < 2 || n_mag > 4097) return b2d::fail(B2D_ERR_SHAPE, "dft_tables: n_mag=%d out of range", n_mag);
    if ((reinterpret_cast<uintptr_t>(dft_tables) & 255u) != 0) return b2d::fail(B2D_ERR_ALIGN, "dft_tables: buffer must be 256-byte aligned");
    dft_tables_kernel<<<b2d::num_sms() * 2, 256, 0, (cudaStream_t)stream>>>(n_mag, dft_tables);
    int rc = b2d::check_launch("dft_tables");
    if (rc) return rc;
    float* img = reinterpret_cast<float*>(reinterpret_cast<char*>(dft_tables) + b2d::cc_table_bytes(n_mag));
    return b2d::dft_image_launch(n_mag, img, (cudaStream_t)stream);
}

extern "C" int b2d_ir_build(const float* c, int64_t ctrl_stride, int mode, const float* f0_frames,
                            const float* dft_tables, int B, int n_frames, int n_mag, double sampling_rate,
                            float* ir, void* stream) {
    if (!c || !dft_tables || !ir) return b2d::fail(B2D_ERR_NULL, "ir_build: null pointer");
    if (mode == B2D_IR_MAG_DYNAMIC && !f0_frames) return b2d::fail(B2D_ERR_NULL, "ir_build: dynamic window needs f0");
    if (B <= 0 || n_frames <= 0 || n_mag < 2 || ctrl_stride < n_mag)
        return b2d::fail(B2D_ERR_SHAPE, "ir_build: bad shape B=%d nF=%d n_mag=%d stride=%lld", B, n_frames, n_mag,
                         (long long)ctrl_stride);
    if (n_mag > 1025) return b2d::fail(B2D_ERR_UNSUPPORTED, "ir_build: n_mag %d > 1025", n_mag);
    IrParams p;
    p.c = c; p.ctrl_stride = ctrl_stride; p.f0 = f0_frames; p.tab = dft_tables;
    p.n_total = B * n_frames; p.M = n_mag;
    p.hw_num = 1.5f * (float)sampling_rate;
    p.ir = ir;
    cudaStream_t st = (cudaStream_t)stream;
    if (mode != B2D_IR_ALLPASS && mode != B2D_IR_MAG_HANN && mode != B2D_IR_MAG_DYNAMIC)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "ir_build: unknown mode %d", mode);
    {
        const int impl = b2d::g_ir_impl.load(std::memory_order_relaxed);
        const bool ok = b2d::ir_tc_supported(mode, n_mag);
        if (impl == 2 && !ok) return b2d::fail(B2D_ERR_UNSUPPORTED, "ir_build: tensor-core path does not support n_mag=%d in mode %d", n_mag, mode);
        if ((impl == 0 || impl == 2) && ok) {
            if ((reinterpret_cast<uintptr_t>(dft_tables) & 255u) != 0) return b2d::fail(B2D_ERR_ALIGN, "ir_build: dft_tables must be 256-byte aligned");
            const float* img = reinterpret_cast<const float*>(reinterpret_cast<const char*>(dft_tables) + b2d::cc_table_bytes(n_mag));
            return b2d::ir_build_tc_launch(c, ctrl_stride, mode, f0_frames, img, B, n_frames, n_mag, sampling_rate, ir, st);
        }
    }
    switch (mode) {
        case B2D_IR_ALLPASS: return launch<B2D_IR_ALLPASS>(p, st);
        case B2D_IR_MAG_HANN: return launch<B2D_IR_MAG_HANN>(p, st);
        case B2D_IR_MAG_DYNAMIC: return launch<B2D_IR_MAG_DYNAMIC>(p, st);
        default: return b2d::fail(B2D_ERR_UNSUPPORTED, "ir_build: unknown mode %d", mode);
    }
}
