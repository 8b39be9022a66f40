// K7: CombSubFast -- STFT-domain filtering of a comb-tooth source and white noise with sqrt-Hann frames.
// Replaces ddsp/vocoder.py:758-784 (the source itself, :743-751 and :764, is b2d_phase_scan + b2d_comb_source).
//
//   frames of N = 2P = 1024 samples at hop P = 512 over the signal zero-padded by P on both sides
//   (frame q covers samples [(q-1)P, (q+1)P), q = 0..nF), analysis and synthesis window sqrt(Hann_N):
//     S_q   = rfft(w * comb_q) * exp(m_h + j pi p_h) + rfft(w * noise_q) * exp(m_n) / 128     (row min(q, nF-1))
//     out   = overlap-add( w * irfft(S_q) ), cropped by P on both sides; no envelope division (w^2 is COLA)
//
// Design.  HBM traffic: 3 x 513 control values per frame = 12 B per output sample, + 4 B comb in and 4 B
// out; everything else stays on chip.  23.4 KB shared memory, 128 registers -> 4 CTAs per SM.
//  * one CTA owns G consecutive hops (G even) of one utterance and walks the G+1 frames that touch them plus the one
//    that completes the last pair, TWO frames per iteration;
//  * per frame one complex 1024-point FFT carries w*(comb + j*noise); both frames of the pair run as a batch
//    through the same three Stockham passes (radix 16, 8, 8), so every pass has >= 128 butterflies for the
//    128 threads;
//  * the two real spectra are separated by conjugate symmetry, filtered, and recombined as Sa + j Sb so that ONE
//    inverse FFT (the forward transform on swapped re/im) returns both real frames -- 1.5 FFTs per frame;
//    torch's C2R convention is kept: the imaginary parts of the DC and Nyquist bins are dropped;
//  * overlap-add needs only the second half of the previous frame: each thread keeps its 4 samples of that tail
//    in registers and writes every hop exactly once with one 128-bit store (deterministic, no atomics).
// The boundary frame of each chunk is recomputed by the neighbouring CTA (G = 32 -> 3 %).
// Noise: explicit samples (parity) or in-kernel Philox uniform in [-1, 1) -- the same stream b2d_ltv_fir draws
// for the same (seed, utterance, sample), so Sins / CombSub / CombSubFast see identical noise.
//
// The derivation is pinned on the CPU by tests/test_csfast_math.py (numpy model with these index formulas).
#ifndef B2D_HOST_EMU               // tests/emu/ runs this kernel's source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif
#include "fft_smem.cuh"

using namespace b2d_fft;
using b2d_fft_smem::kThreads;
using b2d_fft_smem::padi;

namespace {

constexpr int kP = 512;
constexpr int kN = 1024;                                            // transform size: frames of 2 P
constexpr int kPad = b2d_fft_smem::Plan<kN>::kPad, kTw2 = b2d_fft_smem::Plan<kN>::kTw2, kTw3 = b2d_fft_smem::Plan<kN>::kTw3;

struct CfParams {
    const float* comb;         // [B, T]
    const float* noise_in;     // [B, T] or nullptr
    const float* c_hm; const float* c_hp; const float* c_nm;   // [B, nF, P+1] views, frame stride ctrl_stride
    long long ctrl_stride;
    float* out;                // [B, T]
    int nF, G;
    unsigned long long seed;
    long long utt_off;
};

// filter of one bin: Hs = exp(m_h) (cos pi p_h + j sin pi p_h),  Hn = exp(m_n) / 128     (:758,760)
struct BinFilter { float2 hs; float hn; };
__device__ __forceinline__ BinFilter make_filter(float hm, float hp, float nm) {
    float sn, cs;
    sincospif(hp, &sn, &cs);
    const float mag = expf(hm);
    BinFilter f;
    f.hs = make_float2(mag * cs, mag * sn);
    f.hn = expf(nm) * (1.0f / 128.0f);
    return f;
}

constexpr size_t kSmemBytes = (size_t)2 * kPad * sizeof(float2) + (size_t)(kTw2 + kTw3) * sizeof(float2) +
                              (size_t)kN * sizeof(float);      // 17408 + 1920 + 4096 = 23424 B

// PK: the "packed" complex-addition policy (fft_regs.cuh Ar<true>; scalar on Hopper)
template <bool PK>
__global__ void __launch_bounds__(kThreads, 4) combsubfast_kernel(CfParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float2* bufA = reinterpret_cast<float2*>(smem_raw);          // frame a: time -> spectrum -> pair spectrum -> pair time
    float2* bufB = bufA + kPad;                                  // frame b (must follow bufA: batched passes)
    float2* tw2 = bufB + kPad;
    float2* tw3 = tw2 + kTw2;
    float* win = reinterpret_cast<float*>(tw3 + kTw3);           // sqrt(Hann_N), periodic

    const int tid = threadIdx.x;
    const int b = blockIdx.y;
    const int nF = p.nF, T = nF * kP;
    const int h0 = blockIdx.x * p.G, h1 = min(h0 + p.G, nF);
    const float* comb_row = p.comb + (size_t)b * T;
    const float* noise_row = p.noise_in ? p.noise_in + (size_t)b * T : nullptr;
    float* out_row = p.out + (size_t)b * T;
    const unsigned long long utt = (unsigned long long)(p.utt_off + b);

    // ---- one-time tables ----
    for (int i = tid; i < kN; i += kThreads) win[i] = sqrtf(0.5f - 0.5f * cospif((float)i * (2.0f / kN)));
    b2d_fft_smem::init_twiddles<kN>(tw2, tw3, tid);
    __syncthreads();

    // windowed (comb + j noise) of frame q into `buf`; samples outside [0, T) are the zero padding (:766,772)
    auto load_frame = [&](int q, float2* buf) {
#pragma unroll
        for (int u = 0; u < 2; ++u) {
            const int i0 = (tid << 2) + u * (kThreads << 2);     // 4 consecutive in-frame positions
            const int m0 = (q - 1) * kP + i0;                    // multiple of 4; a quad is all inside or all outside
            float4 c = make_float4(0.f, 0.f, 0.f, 0.f), z = c;
            if (m0 >= 0 && m0 < T) {
                c = __ldg(reinterpret_cast<const float4*>(comb_row + m0));
                z = noise_row ? __ldg(reinterpret_cast<const float4*>(noise_row + m0))
                              : b2d::philox_uniform_pm1(p.seed, utt, (uint32_t)(m0 >> 2));
            }
            const float4 w = *reinterpret_cast<const float4*>(win + i0);
            buf[padi(i0 + 0)] = make_float2(w.x * c.x, w.x * z.x);
            buf[padi(i0 + 1)] = make_float2(w.y * c.y, w.y * z.y);
            buf[padi(i0 + 2)] = make_float2(w.z * c.z, w.z * z.z);
            buf[padi(i0 + 3)] = make_float2(w.w * c.w, w.w * z.w);
        }
    };
    // separated + filtered spectrum of one frame at bin k (0 < k < N/2) from Z[k], Z[N-k]
    auto filtered = [](float2 zk, float2 zm, const BinFilter& f) {
        // comb spectrum C = (Z[k] + conj Z[N-k]) / 2, noise spectrum Nz = (Z[k] - conj Z[N-k]) / (2j)
        const float2 C = make_float2(0.5f * (zk.x + zm.x), 0.5f * (zk.y - zm.y));
        const float2 Nz = make_float2(0.5f * (zk.y + zm.y), 0.5f * (zm.x - zk.x));
        float2 s = cmul(C, f.hs);
        s.x = fmaf(Nz.x, f.hn, s.x);
        s.y = fmaf(Nz.y, f.hn, s.y);
        return s;
    };

    float tail[4] = {0.f, 0.f, 0.f, 0.f};      // this thread's 4 samples of the previous frame's second half
    bool have_tail = false;

#pragma unroll 1
    for (int q = h0; q <= h1; q += 2) {
        // frames are always transformed in the same pairs (2m, 2m+1) (G is even): the chunk's last frame h1 is paired with
        // h1 + 1 even though only its first half is used here, so that its round-off does not depend on the chunking and
        // every output sample is bit-identical for any G / batch split.  Frame nF is the last one that exists.
        const bool has_b = q + 1 <= nF;
        const int row_a = min(q, nF - 1), row_b = min(q + 1, nF - 1);            // frame nF reuses row nF-1 (:759,761)
        // ---- controls of both frames for this thread's bins k = tid + 128 u (and k = 0 / 512 on thread 0),
        //      issued before the FFT so their latency hides behind it ----
        float hm_a[4], hp_a[4], nm_a[4], hm_b[4], hp_b[4], nm_b[4];
        const size_t off_a = ((size_t)b * nF + row_a) * (size_t)p.ctrl_stride;
        const size_t off_b = ((size_t)b * nF + row_b) * (size_t)p.ctrl_stride;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int k = tid + u * kThreads;
            hm_a[u] = __ldg(p.c_hm + off_a + k); hp_a[u] = __ldg(p.c_hp + off_a + k); nm_a[u] = __ldg(p.c_nm + off_a + k);
            hm_b[u] = __ldg(p.c_hm + off_b + k); hp_b[u] = __ldg(p.c_hp + off_b + k); nm_b[u] = __ldg(p.c_nm + off_b + k);
        }
        float ny_a[3] = {0.f, 0.f, 0.f}, ny_b[3] = {0.f, 0.f, 0.f};               // Nyquist bin (k = 512), thread 0 only
        if (tid == 0) {
            ny_a[0] = __ldg(p.c_hm + off_a + kP); ny_a[1] = __ldg(p.c_hp + off_a + kP); ny_a[2] = __ldg(p.c_nm + off_a + kP);
            ny_b[0] = __ldg(p.c_hm + off_b + kP); ny_b[1] = __ldg(p.c_hp + off_b + kP); ny_b[2] = __ldg(p.c_nm + off_b + kP);
        }

        // ---- forward: both frames as one batch ----
        load_frame(q, bufA);
        if (has_b) load_frame(q + 1, bufB);
        else {
            for (int i = tid; i < kPad; i += kThreads) bufB[i] = make_float2(0.f, 0.f);
        }
        __syncthreads();
        b2d_fft_smem::fft_forward<1024, 2, PK>(bufA, tw2, tw3, tid);

        // ---- separate, filter, pair: Y = Sa + j Sb (Hermitian extension), stored re/im-swapped in bufA ----
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int k = tid + u * kThreads;
            if (k == 0) continue;                                                 // DC / Nyquist handled below
            const BinFilter fa = make_filter(hm_a[u], hp_a[u], nm_a[u]);
            const BinFilter fb = make_filter(hm_b[u], hp_b[u], nm_b[u]);
            const int ik = padi(k), im = padi(kN - k);
            const float2 sa = filtered(bufA[ik], bufA[im], fa);
            float2 sb = filtered(bufB[ik], bufB[im], fb);
            if (!has_b) sb = make_float2(0.f, 0.f);
            // Y[k] = sa + j sb = (sa.x - sb.y) + j (sa.y + sb.x);  Y[N-k] = conj(sa) + j conj(sb) = (sa.x + sb.y) + j (sb.x - sa.y)
            bufA[ik] = make_float2(sa.y + sb.x, sa.x - sb.y);                     // swapped: (im, re)
            bufA[im] = make_float2(sb.x - sa.y, sa.x + sb.y);
        }
        if (tid == 0) {
            // k = 0 and k = N/2: Z is its own partner; C = Re Z, Nz = Im Z; C2R drops the imaginary part of S
            const BinFilter f0a = make_filter(hm_a[0], hp_a[0], nm_a[0]), f0b = make_filter(hm_b[0], hp_b[0], nm_b[0]);
            const BinFilter fNa = make_filter(ny_a[0], ny_a[1], ny_a[2]), fNb = make_filter(ny_b[0], ny_b[1], ny_b[2]);
            const float2 za0 = bufA[padi(0)], zb0 = bufB[padi(0)], zaN = bufA[padi(kP)], zbN = bufB[padi(kP)];
            const float sa0 = fmaf(za0.y, f0a.hn, za0.x * f0a.hs.x), saN = fmaf(zaN.y, fNa.hn, zaN.x * fNa.hs.x);
            float sb0 = fmaf(zb0.y, f0b.hn, zb0.x * f0b.hs.x), sbN = fmaf(zbN.y, fNb.hn, zbN.x * fNb.hs.x);
            if (!has_b) { sb0 = 0.f; sbN = 0.f; }
            bufA[padi(0)] = make_float2(sb0, sa0);                                // Y = sa + j sb, swapped
            bufA[padi(kP)] = make_float2(sbN, saN);
        }
        __syncthreads();

        // ---- inverse of the pair: ifft(Y) = swap(fft(swap(Y))) / N ----
        b2d_fft_smem::fft_forward<1024, 1, PK>(bufA, tw2, tw3, tid);

        // ---- window, overlap-add, store: frame a = stored .y, frame b = stored .x ----
        const int i0 = tid << 2;
        const float4 w_lo = *reinterpret_cast<const float4*>(win + i0);
        const float4 w_hi = *reinterpret_cast<const float4*>(win + kP + i0);
        const float wl[4] = {w_lo.x, w_lo.y, w_lo.z, w_lo.w}, wh[4] = {w_hi.x, w_hi.y, w_hi.z, w_hi.w};
        float head_a[4], second_a[4], head_b[4], second_b[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 lo = bufA[padi(i0 + e)], hi = bufA[padi(kP + i0 + e)];
            const float sl = wl[e] * (1.0f / kN), sh = wh[e] * (1.0f / kN);
            head_a[e] = lo.y * sl; second_a[e] = hi.y * sh;
            head_b[e] = lo.x * sl; second_b[e] = hi.x * sh;
        }
        if (have_tail)                                                            // hop q-1 = tail(q-1) + head(q)
            b2d::st_global_v4(out_row + (size_t)(q - 1) * kP + i0,
                              make_float4(tail[0] + head_a[0], tail[1] + head_a[1], tail[2] + head_a[2], tail[3] + head_a[3]));
        if (has_b && q < h1) {                                                    // hop q = second(q) + head(q+1)
            b2d::st_global_v4(out_row + (size_t)q * kP + i0,
                              make_float4(second_a[0] + head_b[0], second_a[1] + head_b[1], second_a[2] + head_b[2],
                                          second_a[3] + head_b[3]));
#pragma unroll
            for (int e = 0; e < 4; ++e) tail[e] = second_b[e];
            have_tail = true;
        }
        __syncthreads();                                                          // bufA / bufB are rewritten next iteration
    }
}

}  // namespace

#ifndef B2D_HOST_EMU
extern "C" int b2d_combsubfast_filter(const float* comb, const float* c_harmonic_magnitude, const float* c_harmonic_phase,
                                      const float* c_noise_magnitude, int64_t ctrl_stride, const float* noise_in,
                                      uint64_t seed, int64_t utterance_offset, int B, int n_frames, int block,
                                      float* signal, void* stream) {
    if (!comb || !c_harmonic_magnitude || !c_harmonic_phase || !c_noise_magnitude || !signal)
        return b2d::fail(B2D_ERR_NULL, "combsubfast: null pointer");
    if (B <= 0 || n_frames <= 0) return b2d::fail(B2D_ERR_SHAPE, "combsubfast: bad shape");
    if (block != kP) return b2d::fail(B2D_ERR_UNSUPPORTED, "combsubfast: block size %d (this build: %d)", block, kP);
    if (ctrl_stride < kP + 1) return b2d::fail(B2D_ERR_SHAPE, "combsubfast: control stride %lld < %d", (long long)ctrl_stride, kP + 1);
    if (B > 65535) return b2d::fail(B2D_ERR_UNSUPPORTED, "combsubfast: batch %d > 65535", B);
    if (!b2d::aligned16(comb) || !b2d::aligned16(signal) || (noise_in && !b2d::aligned16(noise_in)))
        return b2d::fail(B2D_ERR_ALIGN, "combsubfast: comb / noise_in / signal must be 16-byte aligned");
    CfParams p;
    p.comb = comb; p.noise_in = noise_in;
    p.c_hm = c_harmonic_magnitude; p.c_hp = c_harmonic_phase; p.c_nm = c_noise_magnitude;
    p.ctrl_stride = ctrl_stride; p.out = signal; p.nF = n_frames;
    int G = 32;            // hops per CTA: shorter chunks when the launch would not fill the GPU (cf. ltv_fir_fft.cu)
    while (G > 2 && (long long)B * ((n_frames + G - 1) / G) < (long long)b2d::num_sms() * 2) G >>= 1;
    p.G = G;
    p.seed = seed; p.utt_off = utterance_offset;
    const dim3 grid((unsigned)((n_frames + p.G - 1) / p.G), B);
    if (b2d::g_fft_packed.load(std::memory_order_relaxed)) combsubfast_kernel<true><<<grid, kThreads, kSmemBytes, (cudaStream_t)stream>>>(p);
    else combsubfast_kernel<false><<<grid, kThreads, kSmemBytes, (cudaStream_t)stream>>>(p);
    return b2d::check_launch("combsubfast");
}
#endif  // B2D_HOST_EMU
