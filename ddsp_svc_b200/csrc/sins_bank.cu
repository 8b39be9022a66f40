// K2: additive sinusoid bank  (reference ddsp/vocoder.py:580,585-594 + ddsp/core.py:66-77).
//
//   sinusoids[t] = sum_{h=1..H} sin(h * phase[t]) * ((1-j/P) A[k,h] + (j/P) A[k+1,h]),  t = kP + j
//
// Mapping: one CTA owns a chunk of consecutive frames of ONE utterance.  The raw
// amplitude rows of the chunk are staged to shared memory by 1-D bulk async copies (TMA,
// UBLKCP) tracked by an mbarrier; exp()/128 and the Nyquist mask are applied once per frame
// there.  Lanes own consecutive samples (4 per thread -> one 128-bit coalesced store), and
// loop over harmonics with the activated amplitudes read as warp-broadcast float4s, so no
// cross-lane reduction is needed.
//
// The kernel is MUFU (sin/cos SFU) bound, so the harmonic set is factored as
//   h = a + 16 b,  a = 1..16 (anchors), b = 0..7 (bases):
//   sin(h p) = sin(a p) cos(16 b p) + cos(a p) sin(16 b p)
// which needs 2 MUFU per anchor + 2 per base (46 per sample for H = 128 instead of 128; the first
// version used 32 anchors x 4 bases = 70 and was SFU bound at 0.31 ms) and 3 FP32 ops per harmonic:
//   amp = fma(dA, frac, A);  P_b += sin(a p) * amp;  Q_b += cos(a p) * amp;
// result = sum_b P_b cos(16 b p) + Q_b sin(16 b p).
//
// The per-sample phase is evaluated in fp64 from the frame-rate scan (phase_scan.cu):
//   x = S_k + ((j+1) f_k + (f_{k+1}-f_k) j (j+1) / (2P)) / sr,  wrapped, rounded to fp32,
// exactly the quantity the reference obtains from its fp64 cumsum (ddsp/vocoder.py:566-572).
#include "b2d_common.cuh"
#include "sins_bank_math.cuh"

using namespace b2d_bank;

namespace {

constexpr int kThreads = 128;
constexpr int kFramesPerCta = 8;

template <int NB, bool MULTI>
__global__ void __launch_bounds__(kThreads, 4) sins_bank_kernel(BankParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int b = blockIdx.y;
    const int k0 = blockIdx.x * kFramesPerCta;
    const int nfr = min(kFramesPerCta, p.nF - k0);  // frames in this chunk
    const int nrows = nfr + 1;                       // amplitude rows k0 .. k0+nfr (clamped)
    const int G = (p.H + kGroup - 1) / kGroup;
    const int HP = G * kGroup;                       // padded row length
    const int Hraw = (p.H + 3) & ~3;

    float* act = reinterpret_cast<float*>(smem_raw);                   // [kF+1][HP]
    float* dlt = act + (kFramesPerCta + 1) * HP;                       // [kF][HP]
    float* raw = dlt + kFramesPerCta * HP;                             // [kF+1][Hraw]
    double* Ss = reinterpret_cast<double*>(raw + (kFramesPerCta + 1) * Hraw);  // [kF]
    float* f0s = reinterpret_cast<float*>(Ss + kFramesPerCta);         // [kF+1]
    __shared__ __align__(8) uint64_t bar;

    const int tid = threadIdx.x;
    const float* crow0 = p.c_amp + ((size_t)b * p.nF) * p.ctrl_stride;

    if (p.use_tma) {
        if (tid == 0) {
            b2d::mbar_init(&bar, 1);
            b2d::fence_mbar_init();
            b2d::mbar_arrive_expect_tx(&bar, (uint32_t)(nrows * Hraw * 4));
            for (int r = 0; r < nrows; ++r) {
                const int k = min(k0 + r, p.nF - 1);
                b2d::tma_load_1d(raw + r * Hraw, crow0 + (size_t)k * p.ctrl_stride, (uint32_t)(Hraw * 4), &bar);
            }
        }
    } else {
        for (int i = tid; i < nrows * p.H; i += kThreads) {
            const int r = i / p.H, h = i - r * p.H;
            const int k = min(k0 + r, p.nF - 1);
            raw[r * Hraw + h] = crow0[(size_t)k * p.ctrl_stride + h];
        }
    }
    for (int r = tid; r < nrows; r += kThreads) {
        const int k = min(k0 + r, p.nF - 1);
        f0s[r] = p.f0[(size_t)b * p.nF + k];
        if (r < nfr) Ss[r] = p.frame_phase[(size_t)b * p.nF + k0 + r];
    }
    __syncthreads();                       // mbarrier init + f0s visible
    if (p.use_tma) b2d::mbar_wait(&bar, 0);

    // activation at frame rate: A = exp(c)/128 * (1[f0*h < sr/2] + 1e-7)   (vocoder.py:580,585)
    for (int i = tid; i < nrows * HP; i += kThreads) {
        const int r = i / HP, hh = i - r * HP;
        float v = 0.f;
        if (hh < p.H) {
            const float c = raw[r * Hraw + hh];
            const float keep = ((f0s[r] * (float)(hh + 1)) < p.nyquist ? 1.0f : 0.0f) + 1e-7f;
            v = (expf(c) * 0.0078125f) * keep;
        }
        act[r * HP + slot_of(hh)] = v;
    }
    __syncthreads();
    for (int i = tid; i < nfr * HP; i += kThreads) dlt[i] = act[i + HP] - act[i];
    __syncthreads();

    const int P = p.P;
    const int quads = (nfr * P) >> 2;
    const float invP = 1.0f / (float)P;
    const double inv2P = 0.5 / (double)P;
    float* out = p.out + (size_t)b * p.nF * P + (size_t)k0 * P;

    for (int q = tid; q < quads; q += kThreads) {
        const int off = q << 2;
        const int r = off / P, j = off - r * P;
        const double fk = (double)f0s[r], dk = (double)f0s[r + 1] - fk, S = Ss[r];
        float x32[4], phase[4], frac[4], acc[4];
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            const double jj = (double)(j + s);
            double x = S + ((jj + 1.0) * fk + dk * (jj * (jj + 1.0)) * inv2P) * p.inv_sr;
            if (p.round_fp32) x = (double)(float)x;
            x -= rint(x);
            x32[s] = (float)x;
            phase[s] = x32[s] * B2D_TWO_PI_F;
            frac[s] = (float)(j + s) * invP;
            acc[s] = 0.f;
        }
        const float* arow = act + r * HP;
        const float* drow = dlt + r * HP;
        if (!MULTI) {
            bank_group<NB, true>(arow, drow, 0, x32, phase, frac, acc);
        } else {
            bank_group<kNBmax, true>(arow, drow, 0, x32, phase, frac, acc);
            for (int g = 1; g < G; ++g) bank_group<kNBmax, false>(arow, drow, g, x32, phase, frac, acc);
        }
        b2d::st_global_v4(out + off, make_float4(acc[0], acc[1], acc[2], acc[3]));
    }
}

template <int NB, bool MULTI>
int launch(const BankParams& p, int B, size_t smem, cudaStream_t st) {
    auto kern = sins_bank_kernel<NB, MULTI>;
    if (smem > 48 * 1024) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return b2d::fail((int)e, "sins_bank: smem attr: %s", cudaGetErrorString(e));
    }
    dim3 grid((p.nF + kFramesPerCta - 1) / kFramesPerCta, B);
    kern<<<grid, kThreads, smem, st>>>(p);
    return b2d::check_launch("sins_bank");
}

}  // namespace

extern "C" int b2d_sins_bank(const float* f0_frames, const double* frame_phase, const float* c_amp,
                             int64_t ctrl_stride, int B, int n_frames, int block, int n_harmonics,
                             double sampling_rate, int round_fp32, float* sinusoids, void* stream) {
    if (!f0_frames || !frame_phase || !c_amp || !sinusoids) return b2d::fail(B2D_ERR_NULL, "sins_bank: null pointer");
    if (B <= 0 || n_frames <= 0 || block <= 0 || n_harmonics <= 0 || ctrl_stride < n_harmonics)
        return b2d::fail(B2D_ERR_SHAPE, "sins_bank: bad shape B=%d nF=%d block=%d H=%d stride=%lld", B, n_frames,
                         block, n_harmonics, (long long)ctrl_stride);
    if (block % 4 != 0) return b2d::fail(B2D_ERR_UNSUPPORTED, "sins_bank: block size %d must be a multiple of 4", block);
    if (n_harmonics > 512) return b2d::fail(B2D_ERR_UNSUPPORTED, "sins_bank: n_harmonics %d > 512", n_harmonics);
    if (B > 65535) return b2d::fail(B2D_ERR_UNSUPPORTED, "sins_bank: batch %d > 65535", B);
    if (!b2d::aligned16(sinusoids)) return b2d::fail(B2D_ERR_ALIGN, "sins_bank: output must be 16-byte aligned");

    BankParams p;
    p.f0 = f0_frames; p.frame_phase = frame_phase; p.c_amp = c_amp; p.ctrl_stride = ctrl_stride;
    p.nF = n_frames; p.P = block; p.H = n_harmonics;
    p.inv_sr = 1.0 / sampling_rate;
    p.nyquist = (float)(sampling_rate / 2.0);
    p.round_fp32 = round_fp32;
    // bulk async copies need 16-byte aligned rows of a 16-byte multiple
    p.use_tma = (n_harmonics % 4 == 0) && b2d::aligned16(c_amp) && (ctrl_stride % 4 == 0);
    p.out = sinusoids;

    const int G = (n_harmonics + kGroup - 1) / kGroup, HP = G * kGroup, Hraw = (n_harmonics + 3) & ~3;
    const size_t smem = (size_t)((kFramesPerCta + 1) * HP + kFramesPerCta * HP + (kFramesPerCta + 1) * Hraw) * 4 +
                        kFramesPerCta * 8 + (kFramesPerCta + 1) * 4 + 16;
    cudaStream_t st = (cudaStream_t)stream;
    if (G > 1) return launch<kNBmax, true>(p, B, smem, st);
    const int nb = (n_harmonics + kNA - 1) / kNA;
    switch (nb) {
        case 1: return launch<1, false>(p, B, smem, st);
        case 2: return launch<2, false>(p, B, smem, st);
        case 3: return launch<3, false>(p, B, smem, st);
        case 4: return launch<4, false>(p, B, smem, st);
        case 5: return launch<5, false>(p, B, smem, st);
        case 6: return launch<6, false>(p, B, smem, st);
        case 7: return launch<7, false>(p, B, smem, st);
        default: return launch<8, false>(p, B, smem, st);
    }
}
