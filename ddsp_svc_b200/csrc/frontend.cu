// Caller-side prologue / epilogue of the synthesis path (SURVEY 8f rank 2): the streaming operations the reference's
// inference drivers run on the CPU (numpy) or as separate eager ops right before and after `model(...)`:
//
//   * Volume_Extractor.extract        ddsp/vocoder.py:147-157   frame RMS of the input audio (reflect-padded, hop windows)
//   * silence mask                    main.py:210-214           threshold, 4-frame edge padding, 9-frame max (dilation)
//   * mask upsample x multiply        main.py:215,260           `seg_output *= upsample(mask, block)` (ddsp/core.py:66-70)
//   * segment cross-fade              main.py:142-149           linear fade over the overlap of two rendered segments
//   * Slicer's frame RMS              slicer.py (main.py:124)   librosa.feature.rms(center=True, constant padding), fp64
//   * segment placement               main.py:266-273           one segment into the whole-file result, faded in place
//
// All are HBM-bound, one pass, coalesced 128-bit accesses where alignment allows; algorithmic bytes: volume 4 B per input
// sample read, mask-apply 8 B per sample (read + write in place), cross-fade 12 B per overlapped sample, slicer RMS
// 4 B per sample per overlapping frame (frame_length / hop of them), placement 8 B per segment sample (+4 B faded).
// No atomics: every output has one writer and a fixed summation order, so results are bit-identical run to run.
#ifndef B2D_HOST_EMU               // tests/emu/ runs these kernels' source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif

namespace {

__device__ __forceinline__ int reflect(int i, int n) {      // numpy.pad(mode='reflect') index (no edge repeat), any offset
    if (n == 1) return 0;
    const int period = 2 * (n - 1);
    i %= period;
    if (i < 0) i += period;
    return i < n ? i : period - i;
}

// one warp per frame: volume[n] = sqrt(mean_{i < hop} pad(audio^2)[n hop + i]),  pad = reflect by (hop/2, (hop+1)/2)
__global__ void __launch_bounds__(256) volume_extract_kernel(const float* __restrict__ audio, int T, int hop, int n_frames,
                                                             float* __restrict__ volume) {
    const int b = blockIdx.y;
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (n >= n_frames) return;
    const float* a = audio + (size_t)b * T;
    const int start = n * hop - hop / 2;                  // index into the unpadded signal of the window's first sample
    // the padded signal has T + hop samples; the reference's last window may be cut short by the slice (numpy clips)
    const int len = min(hop, T + hop - n * hop);
    double acc = 0.0;                                     // numpy sums float32 pairwise; fp64 here is at least as accurate
    for (int i = lane; i < len; i += 32) {
        const int src = start + i;
        const float v = a[(src >= 0 && src < T) ? src : reflect(src, T)];
        acc += (double)(v * v);                           // audio ** 2 is rounded to fp32 first, like the reference
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
    if (lane == 0) volume[(size_t)b * n_frames + n] = sqrtf((float)(acc / (double)len));
}

// mask[n] = max_{|d| <= 4} (volume[clamp(n + d)] > thr)      (main.py:211-213: edge-pad by 4, 9-frame running max)
__global__ void volume_mask_kernel(const float* __restrict__ volume, int n_frames, float thr, float* __restrict__ mask) {
    const int b = blockIdx.y;
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= n_frames) return;
    const float* v = volume + (size_t)b * n_frames;
    float m = 0.f;
#pragma unroll
    for (int d = -4; d <= 4; ++d) m = fmaxf(m, v[min(max(n + d, 0), n_frames - 1)] > thr ? 1.f : 0.f);
    mask[(size_t)b * n_frames + n] = m;
}

// signal[b, t] *= upsample(mask, P)[frame0 P + t]   in place.  The weight reproduces torch's upsample_linear1d with
// align_corners=True on the nF+1 frame values (last one repeated, ddsp/core.py:68) operation by operation: scale =
// float(nF) / float(nF P), src = scale * float(t_global), i0 = floor(src), lambda = src - i0, w = (1-lambda) m[i0] + lambda m[i1].
// For power-of-two block sizes lambda is exactly j/P; for others (441, ...) it carries torch's fp32 rounding of src.
__device__ __forceinline__ float mask_weight(const float* __restrict__ m, int nF_mask, float scale, long long tg) {
    const float src = scale * (float)tg;
    int i0 = (int)floorf(src);
    i0 = min(i0, nF_mask);                                   // input has nF_mask + 1 points
    const float lam = fminf(fmaxf(src - (float)i0, 0.f), 1.f);
    const int i1 = i0 + (i0 < nF_mask ? 1 : 0);
    const float v0 = m[min(i0, nF_mask - 1)], v1 = m[min(i1, nF_mask - 1)];
    // torch's CPU kernel evaluates w0 * v0 + w1 * v1 as fma(w0, v0, w1 * v1) (checked bit for bit on general frame values in
    // tests/test_oracle_frontend.py); written out so the result does not depend on the compiler's contraction choice
    return fmaf(1.f - lam, v0, __fmul_rn(lam, v1));
}

template <bool VEC>
__global__ void __launch_bounds__(256) mask_apply_kernel(float* __restrict__ signal, const float* __restrict__ mask,
                                                         int nF_mask, int frame0, int nF_sig, int P) {
    const int b = blockIdx.y;
    const size_t T = (size_t)nF_sig * P;
    const float* m = mask + (size_t)b * nF_mask;
    float* s = signal + (size_t)b * T;
    const float scale = (float)nF_mask / (float)((long long)nF_mask * P);
    const long long t0 = (long long)frame0 * P;
    if (VEC) {
        for (size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q < T / 4; q += (size_t)gridDim.x * blockDim.x) {
            const size_t t = q * 4;
            float4 v = *reinterpret_cast<const float4*>(s + t);
            v.x *= mask_weight(m, nF_mask, scale, t0 + (long long)t);
            v.y *= mask_weight(m, nF_mask, scale, t0 + (long long)t + 1);
            v.z *= mask_weight(m, nF_mask, scale, t0 + (long long)t + 2);
            v.w *= mask_weight(m, nF_mask, scale, t0 + (long long)t + 3);
            *reinterpret_cast<float4*>(s + t) = v;
        }
    } else {
        for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < T; t += (size_t)gridDim.x * blockDim.x)
            s[t] *= mask_weight(m, nF_mask, scale, t0 + (long long)t);
    }
}

// sample r < fade of main.py:147's fade, (1 - k_r) a + k_r b in fp64 rounded to fp32, k = numpy.linspace(0, 1, fade):
// k_r = r * step with step = 1 / (fade - 1) (the caller's fade_step), the end point pinned to exactly 1, [0] for fade 1
__device__ __forceinline__ double fade_step(long long fade) { return fade > 1 ? 1.0 / (double)(fade - 1) : 0.0; }
__device__ __forceinline__ float fade_sample(float a, float b, long long r, long long fade, double step) {
    const double k = (fade == 1) ? 0.0 : (r == fade - 1 ? 1.0 : (double)r * step);   // linspace pins the end point
    return (float)((1.0 - k) * (double)a + k * (double)b);
}

// out = [ a[:idx] | (1-k) a[idx:] + k b[:fade] | b[fade:] ],  fade = len_a - idx,  k = linspace(0, 1, fade)   (main.py:142-149)
__global__ void __launch_bounds__(256) cross_fade_kernel(const float* __restrict__ a, long long len_a, const float* __restrict__ b,
                                                         long long len_b, long long idx, float* __restrict__ out) {
    const long long fade = len_a - idx, total = idx + len_b;
    const double step = fade_step(fade);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        float v;
        if (i < idx) v = a[i];
        else if (i < len_a) {
            const long long r = i - idx;
            v = fade_sample(a[i], b[r], r, fade, step);
        } else v = b[i - idx];
        out[i] = v;
    }
}

// main.py's assembly step for one segment, in place on the whole-file result (zero where nothing was written yet):
// result[idx + r] = fade_sample(result[idx + r], seg[r], r, fade_len) for r < fade_len, = seg[r] after, r < seg_len.
// The samples from idx + seg_len on are left alone: main.py's cross_fade drops nothing there, since fade_len <= seg_len.
__global__ void __launch_bounds__(256) segment_place_kernel(float* __restrict__ result, const float* __restrict__ seg,
                                                            long long seg_len, long long idx, long long fade_len) {
    const double step = fade_step(fade_len);
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < seg_len; r += (long long)gridDim.x * blockDim.x)
        result[idx + r] = r < fade_len ? fade_sample(result[idx + r], seg[r], r, fade_len, step) : seg[r];
}

// warp-wide fp64 sum, butterfly order (every lane ends with the same bits)
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    return v;
}

// librosa.feature.rms(y, frame_length, hop_length) as the reference's Slicer calls it (center=True, constant padding):
// frame f covers y[f hop - frame_length / 2 + j], j < frame_length, zero outside the signal, and
// rms[f] = sqrt(sum_j y^2 / frame_length), squares exact and summed in fp64, rounded to fp32 once.  One warp per frame;
// each lane sums its strided samples in order, then the warp's butterfly: a fixed order, so the result is deterministic.
__global__ void __launch_bounds__(256) slicer_rms_kernel(const float* __restrict__ y, long long n, int frame_length, int hop,
                                                         long long n_frames, float* __restrict__ rms) {
    const long long f = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (f >= n_frames) return;
    const long long start = f * hop - frame_length / 2;
    const long long j0 = start < 0 ? -start : 0, j1 = min((long long)frame_length, n - start);
    double acc = 0.0;
    for (long long j = j0 + lane; j < j1; j += 32) {
        const double v = (double)y[start + j];
        acc += v * v;
    }
    acc = warp_sum(acc);
    if (lane == 0) rms[f] = (float)sqrt(acc / (double)frame_length);
}

}  // namespace

#ifndef B2D_HOST_EMU
extern "C" int b2d_volume_extract(const float* audio, int B, int n_samples, int hop, float* volume, void* stream) {
    if (!audio || !volume) return b2d::fail(B2D_ERR_NULL, "volume_extract: null pointer");
    if (B <= 0 || n_samples < 2 || hop <= 0 || hop / 2 >= n_samples)
        return b2d::fail(B2D_ERR_SHAPE, "volume_extract: bad shape B=%d T=%d hop=%d (reflect padding needs hop/2 < T)", B, n_samples, hop);
    if (B > 65535) return b2d::fail(B2D_ERR_UNSUPPORTED, "volume_extract: batch %d > 65535", B);
    const int n_frames = n_samples / hop + 1;
    dim3 grid((n_frames + 7) / 8, B);
    volume_extract_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(audio, n_samples, hop, n_frames, volume);
    return b2d::check_launch("volume_extract");
}

extern "C" int b2d_volume_mask(const float* volume, int B, int n_frames, float threshold, float* mask, void* stream) {
    if (!volume || !mask) return b2d::fail(B2D_ERR_NULL, "volume_mask: null pointer");
    if (B <= 0 || n_frames <= 0 || B > 65535) return b2d::fail(B2D_ERR_SHAPE, "volume_mask: bad shape B=%d nF=%d", B, n_frames);
    dim3 grid((n_frames + 255) / 256, B);
    volume_mask_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(volume, n_frames, threshold, mask);
    return b2d::check_launch("volume_mask");
}

extern "C" int b2d_mask_apply(float* signal, const float* mask_frames, int B, int n_mask_frames, int frame_offset,
                              int n_frames, int block, void* stream) {
    if (!signal || !mask_frames) return b2d::fail(B2D_ERR_NULL, "mask_apply: null pointer");
    if (B <= 0 || n_frames <= 0 || block <= 0 || n_mask_frames <= 0 || frame_offset < 0 || frame_offset + n_frames > n_mask_frames)
        return b2d::fail(B2D_ERR_SHAPE, "mask_apply: bad shape B=%d frames [%d, %d) of %d, block=%d", B, frame_offset,
                         frame_offset + n_frames, n_mask_frames, block);
    if (B > 65535) return b2d::fail(B2D_ERR_UNSUPPORTED, "mask_apply: batch %d > 65535", B);
    const size_t T = (size_t)n_frames * block;
    const bool vec = (block % 4 == 0) && b2d::aligned16(signal);
    const size_t work = vec ? T / 4 : T;
    unsigned gx = (unsigned)((work + 255) / 256);
    if (gx > (unsigned)b2d::num_sms() * 16u) gx = (unsigned)b2d::num_sms() * 16u;
    if (gx == 0) gx = 1;
    dim3 grid(gx, B);
    if (vec) mask_apply_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(signal, mask_frames, n_mask_frames, frame_offset, n_frames, block);
    else mask_apply_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(signal, mask_frames, n_mask_frames, frame_offset, n_frames, block);
    return b2d::check_launch("mask_apply");
}

extern "C" int b2d_cross_fade(const float* a, int64_t len_a, const float* b, int64_t len_b, int64_t idx, float* out, void* stream) {
    if (!a || !b || !out) return b2d::fail(B2D_ERR_NULL, "cross_fade: null pointer");
    if (len_a <= 0 || len_b <= 0 || idx < 0 || idx >= len_a || len_a - idx > len_b)
        return b2d::fail(B2D_ERR_SHAPE, "cross_fade: need 0 <= idx < len_a and len_a - idx <= len_b (got %lld, %lld, %lld)",
                         (long long)len_a, (long long)len_b, (long long)idx);
    const long long total = idx + len_b;
    long long gx = (total + 255) / 256;
    if (gx > b2d::num_sms() * 16) gx = b2d::num_sms() * 16;
    cross_fade_kernel<<<(unsigned)gx, 256, 0, (cudaStream_t)stream>>>(a, len_a, b, len_b, idx, out);
    return b2d::check_launch("cross_fade");
}

extern "C" int b2d_slicer_rms(const float* audio, int64_t n_samples, int frame_length, int hop, float* rms, void* stream) {
    if (!audio || !rms) return b2d::fail(B2D_ERR_NULL, "slicer_rms: null pointer");
    if (n_samples <= 0 || frame_length <= 0 || hop <= 0)
        return b2d::fail(B2D_ERR_SHAPE, "slicer_rms: bad shape n=%lld frame_length=%d hop=%d", (long long)n_samples,
                         frame_length, hop);
    const long long padded = (long long)n_samples + 2 * (frame_length / 2);
    if (padded < frame_length)
        return b2d::fail(B2D_ERR_SHAPE, "slicer_rms: %lld samples padded by %d each side are shorter than one frame of %d",
                         (long long)n_samples, frame_length / 2, frame_length);
    const long long n_frames = 1 + (padded - frame_length) / hop;
    const long long blocks = (n_frames + 7) / 8;
    if (blocks > 0x7fffffffLL) return b2d::fail(B2D_ERR_UNSUPPORTED, "slicer_rms: %lld frames", n_frames);
    slicer_rms_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(audio, n_samples, frame_length, hop, n_frames, rms);
    return b2d::check_launch("slicer_rms");
}

extern "C" int b2d_segment_place(float* result, int64_t result_len, const float* seg, int64_t seg_len, int64_t idx,
                                 int64_t fade_len, void* stream) {
    if (!result || !seg) return b2d::fail(B2D_ERR_NULL, "segment_place: null pointer");
    if (seg_len <= 0 || idx < 0 || fade_len < 0 || fade_len > seg_len || idx + seg_len > result_len)
        return b2d::fail(B2D_ERR_SHAPE, "segment_place: need idx >= 0, 0 <= fade_len <= seg_len and idx + seg_len <= "
                         "result_len (got idx %lld, fade_len %lld, seg_len %lld, result_len %lld)", (long long)idx,
                         (long long)fade_len, (long long)seg_len, (long long)result_len);
    long long gx = (seg_len + 255) / 256;
    if (gx > b2d::num_sms() * 16) gx = b2d::num_sms() * 16;
    segment_place_kernel<<<(unsigned)gx, 256, 0, (cudaStream_t)stream>>>(result, seg, seg_len, idx, fade_len);
    return b2d::check_launch("segment_place");
}
#endif  // B2D_HOST_EMU
