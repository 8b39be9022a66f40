// Real-time conversion block of gui.py on the device: f0 regridding, the SOLA shift search and the crossfade.
//
//   rt_regrid     np.interp between two uniform grids in one CTA, positions and values in fp64 as numpy computes them
//                 (slope (y1 - y0) / (x1 - x0), then slope (x - x0) + y0, no fused multiply-add), values held at the
//                 edges.  mode 0 (Enhancer.enhance, enhancer.py:65-70): src scaled by real_factor in fp32, regridded.
//                 mode 1 (F0_Extractor 'rmvpe' + uv_interp, ddsp/vocoder.py:108-118 and :138-144): unvoiced src frames
//                 filled from their voiced neighbours (rounded to fp32, as numpy stores them into the fp32 array),
//                 f0 and the uv flag regridded, frames with interpolated uv > 0.5 zeroed, `pad` leading zero frames,
//                 then the fp64 second fill, the clamp to f0_min, and the fp32 pitch factor.  "No voiced frame" skips a
//                 fill, as the reference's `len(f0[~uv]) > 0` guard does.  The neighbour search is a CTA-wide max-scan
//                 in chunks of kRegridThreads, so any length runs in one launch.
//   rt_sola       gui.py:434-440: score[s] = sum_k x[s + k] buf[k] / sqrt(sum_k x[s + k]^2 + 1e-8), s in [0, search],
//                 and the first index of the largest score (torch.argmax) written to device memory.  One CTA, one warp
//                 per shift.
//   rt_pv_bins    phase_vocoder's analysis (gui.py:15-31): direct rfft bins of a w and b w, w = sqrt(fade_out fade_in),
//                 one warp per bin; the twiddle angle is reduced as (k m) mod n in integers.  Writes |fa| + |fb| (doubled
//                 off DC / Nyquist), angle(fa) / pi and the wrapped phase difference / pi.
//   rt_crossfade  y[t] = x[shift + t] for t < block + crossfade, its first `crossfade` samples replaced by the sin^2
//                 linear fade (gui.py:451-452, fp32 in torch's order) or by phase_vocoder's direct synthesis sum
//                 (cospif of 2 ((k t) mod n) / n + dphi t / n + phia).  out = y[:block], next_buf = y[block:].
//
// No atomics: every output has one writer and a fixed summation order, so results are bit-identical run to run.
#include <climits>
#ifndef B2D_HOST_EMU               // tests/emu/ runs these kernels' source on the CPU (host_emu.h provides the shims)
#include "b2d_common.cuh"
#endif

namespace {

constexpr int kRegridThreads = 256;
constexpr int kSolaThreads = 1024;
constexpr int kCrossfadeThreads = 256;
constexpr int kMaxCrossfade = 32768;   // (k t) stays below 2^31

// fp64 arithmetic without contraction into fma, as numpy's interp computes it
#ifdef B2D_HOST_EMU
inline double dmul(double a, double b) { return a * b; }
inline double dadd(double a, double b) { return a + b; }
inline double ddiv(double a, double b) { return a / b; }
#else
__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
#endif

struct RtRegridParams {
    const float* src;              // [n_src]
    int n_src;
    double src_step, src_div;      // source position i: (src_step i) / src_div
    float src_scale;               // mode 0: src values times src_scale in fp32
    int n_dst, pad;                // output frames; the first `pad` are zero, the rest regridded from position 0
    double dst_step;               // target position j - pad: dst_step (j - pad)
    int mode;                      // 0 plain, 1 rmvpe post-processing
    double f0_min;                 // mode 1: clamp
    float post_scale;              // mode 1: fp32 factor applied last (pitch_adjust)
    float* out;                    // [n_dst]
    double* vsrc;                  // workspace [n_src]
    double* vdst;                  // workspace [n_dst]
    int* prev;                     // workspace [max(n_src, n_dst)]
};

__device__ __forceinline__ double src_pos(const RtRegridParams& p, int i) {
    return ddiv(dmul(p.src_step, (double)i), p.src_div);
}

// np.interp(x, positions, y(i)) over the source grid (x >= 0 = position 0), the right edge held at y(n - 1)
template <class Y>
__device__ double interp_src(const RtRegridParams& p, Y y, double x) {
    const int n = p.n_src;
    if (n == 1 || x >= src_pos(p, n - 1)) return y(n - 1);
    int i = (int)floor(x * p.src_div / p.src_step);          // a guess, corrected against the exact positions
    i = min(max(i, 0), n - 2);
    while (i > 0 && src_pos(p, i) > x) --i;
    while (i < n - 2 && src_pos(p, i + 1) <= x) ++i;
    const double x0 = src_pos(p, i), y0 = y(i);
    if (x0 == x) return y0;
    const double slope = ddiv(y(i + 1) - y0, src_pos(p, i + 1) - x0);
    return dadd(dmul(slope, x - x0), y0);
}

// inclusive max-scan over the CTA; *total = the chunk's maximum.  Starts and ends with the CTA converged.
__device__ int scan_max(int v, int* total, int (&s)[2][kRegridThreads]) {
    const int t = threadIdx.x;
    int cur = 0;
    s[0][t] = v;
    __syncthreads();
    for (int off = 1; off < kRegridThreads; off <<= 1) {
        int x = s[cur][t];
        if (t >= off) x = max(x, s[cur][t - off]);
        s[cur ^ 1][t] = x;
        cur ^= 1;
        __syncthreads();
    }
    const int r = s[cur][t];
    *total = s[cur][kRegridThreads - 1];
    __syncthreads();
    return r;
}

// np.interp(where(uv), where(~uv), v[~uv]) stored into v[uv], uv = (v == 0); every voiced value is left as it is, so
// reads of neighbours never meet a write.  round_f32: the stored value is rounded to fp32 (an fp32 array).
__device__ void fill_unvoiced(double* v, int n, int* prev, bool round_f32, int (&s)[2][kRegridThreads]) {
    const int t = threadIdx.x;
    int carry = -1, total;
    for (int base = 0; base < n; base += kRegridThreads) {
        const int i = base + t;
        const int r = scan_max(i < n && v[i] != 0.0 ? i : -1, &total, s);
        if (i < n) prev[i] = max(r, carry);
        carry = max(carry, total);
    }
    if (carry < 0) return;                                   // no voiced frame (uniform over the CTA)
    int next_carry = INT_MAX;
    for (int hi = n - 1; hi >= 0; hi -= kRegridThreads) {
        const int i = hi - t;                                // thread order runs down the indices
        const bool voiced = i >= 0 && v[i] != 0.0;
        const int r = scan_max(voiced ? -i : INT_MIN, &total, s);
        const int q = min(r == INT_MIN ? INT_MAX : -r, next_carry);
        if (total != INT_MIN) next_carry = min(next_carry, -total);
        if (i >= 0 && !voiced) {
            const int pv = prev[i];
            double f;
            if (pv < 0) f = v[q];
            else if (q == INT_MAX) f = v[pv];
            else f = dadd(dmul(ddiv(v[q] - v[pv], (double)(q - pv)), (double)(i - pv)), v[pv]);
            v[i] = round_f32 ? (double)(float)f : f;
        }
    }
}

__global__ void __launch_bounds__(kRegridThreads) rt_regrid_kernel(const RtRegridParams p) {
    B2D_SHARED(int, s, [2][kRegridThreads]);
    const int t = threadIdx.x;
    const bool rmvpe = p.mode == 1;
    for (int i = t; i < p.n_src; i += kRegridThreads)
        p.vsrc[i] = rmvpe ? (double)p.src[i] : (double)__fmul_rn(p.src[i], p.src_scale);
    __syncthreads();
    if (rmvpe) {
        fill_unvoiced(p.vsrc, p.n_src, p.prev, true, s);
        __syncthreads();
    }
    for (int j = t; j < p.n_dst; j += kRegridThreads) {
        double f = 0.0;
        if (j >= p.pad) {
            const double x = dmul(p.dst_step, (double)(j - p.pad));
            f = interp_src(p, [&](int i) { return p.vsrc[i]; }, x);
            // the uv flag of the unfilled source, regridded the same way
            if (rmvpe && interp_src(p, [&](int i) { return p.src[i] == 0.f ? 1.0 : 0.0; }, x) > 0.5) f = 0.0;
        }
        if (rmvpe) p.vdst[j] = f;
        else p.out[j] = (float)f;
    }
    if (!rmvpe) return;
    __syncthreads();
    fill_unvoiced(p.vdst, p.n_dst, p.prev, false, s);
    __syncthreads();
    for (int j = t; j < p.n_dst; j += kRegridThreads) {
        double f = p.vdst[j];
        if (f < p.f0_min) f = p.f0_min;
        p.out[j] = __fmul_rn((float)f, p.post_scale);
    }
}

__global__ void __launch_bounds__(kSolaThreads) rt_sola_kernel(const float* __restrict__ x, const float* __restrict__ buf,
                                                             int cf, int search, int* __restrict__ shift) {
    B2D_SHARED(float, best_v, [kSolaThreads / 32]);
    B2D_SHARED(int, best_i, [kSolaThreads / 32]);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float bv = -INFINITY;
    int bi = 0;
    for (int s = warp; s <= search; s += kSolaThreads / 32) {
        float nom = 0.f, den = 0.f;
        for (int k = lane; k < cf; k += 32) {
            const float v = __ldg(x + s + k);
            nom = fmaf(v, __ldg(buf + k), nom);
            den = fmaf(v, v, den);
        }
        for (int off = 16; off; off >>= 1) {
            nom += __shfl_xor_sync(0xffffffffu, nom, off);
            den += __shfl_xor_sync(0xffffffffu, den, off);
        }
        const float score = nom / sqrtf(den + 1e-8f);
        if (score > bv || s == warp) { bv = score; bi = s; }   // shifts rise per warp: keep the first maximum
    }
    if (lane == 0) { best_v[warp] = bv; best_i[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float v = best_v[0];
        int i = best_i[0];
        for (int w = 1; w < kSolaThreads / 32 && w <= search; ++w)
            if (best_v[w] > v || (best_v[w] == v && best_i[w] < i)) { v = best_v[w]; i = best_i[w]; }
        *shift = i;
    }
}

struct RtCrossfadeParams {
    const float* x;                // x[shift + t], t < block + cf
    const int* shift;
    const float* buf;              // [cf] the previous block's tail
    const float* fade_in;          // [cf]
    const float* fade_out;         // [cf]
    int block, cf;
    float* bins;                   // phase vocoder: [3][cf / 2 + 1] (|fa| + |fb| (doubled), phia / pi, dphi / pi)
    float* out;                    // [block]
    float* next_buf;               // [cf]
};

__global__ void __launch_bounds__(kCrossfadeThreads) rt_pv_bins_kernel(const RtCrossfadeParams p) {
    const int lane = threadIdx.x & 31;
    const int k = blockIdx.x * (kCrossfadeThreads / 32) + (threadIdx.x >> 5);
    const int n = p.cf, nb = n / 2 + 1;
    if (k >= nb) return;                                     // whole warps leave together
    const float* b = p.x + *p.shift;
    float ar = 0.f, ai = 0.f, br = 0.f, bi = 0.f;
    for (int m = lane; m < n; m += 32) {
        const float w = sqrtf(__fmul_rn(p.fade_out[m], p.fade_in[m]));
        const int r = (int)(((long long)k * m) % n);
        float sn, cs;
        sincospif(2.f * (float)r / (float)n, &sn, &cs);
        const float aw = p.buf[m] * w, bw = b[m] * w;
        ar = fmaf(aw, cs, ar);
        ai = fmaf(-aw, sn, ai);
        br = fmaf(bw, cs, br);
        bi = fmaf(-bw, sn, bi);
    }
    for (int off = 16; off; off >>= 1) {
        ar += __shfl_xor_sync(0xffffffffu, ar, off);
        ai += __shfl_xor_sync(0xffffffffu, ai, off);
        br += __shfl_xor_sync(0xffffffffu, br, off);
        bi += __shfl_xor_sync(0xffffffffu, bi, off);
    }
    if (lane == 0) {
        float amp = hypotf(ar, ai) + hypotf(br, bi);
        if (k >= 1 && k <= (n - 1) / 2) amp *= 2.f;
        const float pa = atan2f(ai, ar), pb = atan2f(bi, br);
        float d = (pb - pa) / B2D_PI_F;                      // (phib - phia) / pi, wrapped to [-1, 1)
        d -= 2.f * floorf(0.5f * d + 0.5f);
        p.bins[k] = amp;
        p.bins[nb + k] = pa / B2D_PI_F;
        p.bins[2 * nb + k] = d;
    }
}

template <bool PV>
__global__ void __launch_bounds__(kCrossfadeThreads) rt_crossfade_kernel(const RtCrossfadeParams p) {
    const int t = blockIdx.x * kCrossfadeThreads + threadIdx.x;
    if (t >= p.block + p.cf) return;
    const float xv = p.x[*p.shift + t];
    float y = xv;
    if (t < p.cf) {
        const float fi = p.fade_in[t], fo = p.fade_out[t], a = p.buf[t];
        if (PV) {
            const int n = p.cf, nb = n / 2 + 1;
            const float tn = (float)t / (float)n;
            float acc = 0.f;
            for (int k = 0; k < nb; ++k) {
                const int r = (int)(((long long)k * t) % n);
                const float arg = fmaf(__ldg(p.bins + 2 * nb + k), tn, __ldg(p.bins + nb + k)) + 2.f * (float)r / (float)n;
                acc = fmaf(__ldg(p.bins + k), cospif(arg), acc);
            }
            const float w = sqrtf(__fmul_rn(fo, fi));
            y = __fadd_rn(__fadd_rn(__fmul_rn(a, __fmul_rn(fo, fo)), __fmul_rn(xv, __fmul_rn(fi, fi))),
                          __fdiv_rn(__fmul_rn(acc, w), (float)n));
        } else {
            y = __fadd_rn(__fmul_rn(xv, fi), __fmul_rn(a, fo));
        }
    }
    if (t < p.block) p.out[t] = y;
    else p.next_buf[t - p.block] = y;
}

}  // namespace

#ifndef B2D_HOST_EMU
namespace {
size_t regrid_ws_bytes(int n_src, int n_dst) {
    return b2d::align256((size_t)n_src * 8) + b2d::align256((size_t)n_dst * 8) +
           b2d::align256((size_t)(n_src > n_dst ? n_src : n_dst) * 4);
}
}  // namespace

extern "C" size_t b2d_rt_f0_regrid_workspace_bytes(int n_src, int n_dst) {
    return n_src > 0 && n_dst > 0 ? regrid_ws_bytes(n_src, n_dst) : 0;
}

extern "C" int b2d_rt_f0_regrid(const float* src, int n_src, double src_step, double src_div, float src_scale,
                                int n_dst, int pad, double dst_step, int mode, double f0_min, float post_scale,
                                float* out, void* workspace, size_t workspace_bytes, void* stream) {
    if (!src || !out || !workspace) return b2d::fail(B2D_ERR_NULL, "rt_f0_regrid: null pointer");
    if (n_src <= 0 || n_dst <= 0 || pad < 0 || pad > n_dst || !(src_step > 0.0) || !(src_div > 0.0) ||
        !(dst_step > 0.0) || (mode != 0 && mode != 1) || (mode == 0 && pad != 0))
        return b2d::fail(B2D_ERR_SHAPE, "rt_f0_regrid: bad shape or mode");
    if (workspace_bytes < regrid_ws_bytes(n_src, n_dst))
        return b2d::fail(B2D_ERR_WORKSPACE, "rt_f0_regrid: workspace of %zu bytes, need %zu", workspace_bytes,
                         regrid_ws_bytes(n_src, n_dst));
    if (!b2d::aligned16(workspace)) return b2d::fail(B2D_ERR_ALIGN, "rt_f0_regrid: workspace not 16-byte aligned");
    RtRegridParams p{};
    p.src = src; p.n_src = n_src; p.src_step = src_step; p.src_div = src_div; p.src_scale = src_scale;
    p.n_dst = n_dst; p.pad = pad; p.dst_step = dst_step; p.mode = mode; p.f0_min = f0_min; p.post_scale = post_scale;
    p.out = out;
    size_t off = 0;
    p.vsrc = reinterpret_cast<double*>(static_cast<char*>(workspace) + b2d::ws_append(off, 2 * (size_t)n_src));
    p.vdst = reinterpret_cast<double*>(static_cast<char*>(workspace) + b2d::ws_append(off, 2 * (size_t)n_dst));
    p.prev = reinterpret_cast<int*>(static_cast<char*>(workspace) + b2d::ws_append(off, n_src > n_dst ? n_src : n_dst));
    rt_regrid_kernel<<<1, kRegridThreads, 0, (cudaStream_t)stream>>>(p);
    return b2d::check_launch("rt_f0_regrid");
}

extern "C" int b2d_rt_sola(const float* x, const float* buf, int crossfade, int search, int* shift, void* stream) {
    if (!x || !buf || !shift) return b2d::fail(B2D_ERR_NULL, "rt_sola: null pointer");
    if (crossfade <= 0 || search < 0) return b2d::fail(B2D_ERR_SHAPE, "rt_sola: bad shape");
    rt_sola_kernel<<<1, kSolaThreads, 0, (cudaStream_t)stream>>>(x, buf, crossfade, search, shift);
    return b2d::check_launch("rt_sola");
}

extern "C" size_t b2d_rt_crossfade_workspace_bytes(int crossfade, int phase_vocoder) {
    return crossfade > 0 ? (phase_vocoder ? (size_t)3 * (crossfade / 2 + 1) * 4 : 0) : 0;
}

extern "C" int b2d_rt_crossfade(const float* x, const int* shift, const float* buf, const float* fade_in,
                                const float* fade_out, int block, int crossfade, int phase_vocoder, float* out,
                                float* next_buf, void* workspace, size_t workspace_bytes, void* stream) {
    if (!x || !shift || !buf || !fade_in || !fade_out || !out || !next_buf || (phase_vocoder && !workspace))
        return b2d::fail(B2D_ERR_NULL, "rt_crossfade: null pointer");
    if (block <= 0 || crossfade <= 0) return b2d::fail(B2D_ERR_SHAPE, "rt_crossfade: bad shape");
    if (crossfade > kMaxCrossfade)
        return b2d::fail(B2D_ERR_UNSUPPORTED, "rt_crossfade: crossfade %d > %d", crossfade, kMaxCrossfade);
    if (workspace_bytes < b2d_rt_crossfade_workspace_bytes(crossfade, phase_vocoder))
        return b2d::fail(B2D_ERR_WORKSPACE, "rt_crossfade: workspace too small");
    RtCrossfadeParams p{x, shift, buf, fade_in, fade_out, block, crossfade, static_cast<float*>(workspace), out,
                        next_buf};
    const cudaStream_t s = (cudaStream_t)stream;
    const unsigned grid = (unsigned)((block + crossfade + kCrossfadeThreads - 1) / kCrossfadeThreads);
    if (phase_vocoder) {
        const int warps = kCrossfadeThreads / 32;
        rt_pv_bins_kernel<<<(crossfade / 2 + 1 + warps - 1) / warps, kCrossfadeThreads, 0, s>>>(p);
        if (int rc = b2d::check_launch("rt_pv_bins")) return rc;
        rt_crossfade_kernel<true><<<grid, kCrossfadeThreads, 0, s>>>(p);
    } else {
        rt_crossfade_kernel<false><<<grid, kCrossfadeThreads, 0, s>>>(p);
    }
    return b2d::check_launch("rt_crossfade");
}
#endif  // B2D_HOST_EMU
