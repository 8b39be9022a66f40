// Small complex DFTs held in registers: the butterflies of the shared-memory Stockham FFTs in superfast.cu
// (2048 points) and combsubfast.cu (1024 points).
#pragma once
#ifndef B2D_HOST_EMU
#include <cuda_runtime.h>
#endif

namespace b2d_fft {

__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
    return make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ float2 mul_mj(float2 a) { return make_float2(a.y, -a.x); }  // a * (-j)

// Complex add / subtract policy.  PK selects the "packed" instantiation of the FFT kernels (b2d_set_fft_arith); Hopper
// has no packed FP32 add (f32x2 needs sm_100), so both policies are two scalar FADDs and give identical results.
template <bool PK> struct Ar {
    static __device__ __forceinline__ float2 add(float2 a, float2 b) { return cadd(a, b); }
    static __device__ __forceinline__ float2 sub(float2 a, float2 b) { return csub(a, b); }
};

// forward DFT of 2^n points, natural order in and out (recursive decimation in time, unrolled)
template <int R, bool PK = false> struct Dft;
template <bool PK> struct Dft<1, PK> { static __device__ __forceinline__ void run(float2*) {} };
template <bool PK> struct Dft<2, PK> {
    static __device__ __forceinline__ void run(float2* v) {
        const float2 a = v[0], b = v[1];
        v[0] = Ar<PK>::add(a, b); v[1] = Ar<PK>::sub(a, b);
    }
};
template <int R, int K> __device__ __forceinline__ float2 twid(float2 o) {  // o * exp(-2 pi i K / R)
    if (K == 0) return o;
    if (4 * K == R) return mul_mj(o);
    if (8 * K == R) return make_float2(0.70710678118654752f * (o.x + o.y), 0.70710678118654752f * (o.y - o.x));
    if (8 * K == 3 * R) return make_float2(0.70710678118654752f * (o.y - o.x), -0.70710678118654752f * (o.x + o.y));
    // remaining cases: R = 16, K in {1,3,5,7}
    const float c1 = 0.92387953251128674f, s1 = 0.38268343236508977f;
    const float c = (K == 1) ? c1 : (K == 3) ? s1 : (K == 5) ? -s1 : -c1;
    const float s = (K == 1) ? s1 : (K == 3) ? c1 : (K == 5) ? c1 : s1;
    return make_float2(fmaf(o.x, c, o.y * s), fmaf(o.y, c, -o.x * s));  // (c - j s) * o
}
template <int R, int K, bool PK> struct Comb {
    static __device__ __forceinline__ void run(const float2* e, const float2* o, float2* v) {
        const float2 t = twid<R, K>(o[K]);
        v[K] = Ar<PK>::add(e[K], t);
        v[K + R / 2] = Ar<PK>::sub(e[K], t);
        Comb<R, K + 1, PK>::run(e, o, v);
    }
};
template <int R, bool PK> struct Comb<R, R / 2, PK> { static __device__ __forceinline__ void run(const float2*, const float2*, float2*) {} };
template <int R, bool PK> struct Dft {
    static __device__ __forceinline__ void run(float2* v) {
        float2 e[R / 2], o[R / 2];
#pragma unroll
        for (int i = 0; i < R / 2; ++i) { e[i] = v[2 * i]; o[i] = v[2 * i + 1]; }
        Dft<R / 2, PK>::run(e);
        Dft<R / 2, PK>::run(o);
        Comb<R, 0, PK>::run(e, o, v);
    }
};

// 16-point DFT whose inputs 8..15 are zero (the first pass of a transform whose upper half is zero padding):
//   X[2m] = DFT8(v[r])[m],  X[2m+1] = DFT8(v[r] W16^r)[m]     (decimation in frequency with v[r + 8] = 0)
// -- the 16 closing additions of the full butterfly disappear.  Reads v[0..7], writes v[0..15] in natural order.
template <bool PK> struct Dft16ZeroUpper {
    static __device__ __forceinline__ void run(float2* v) {
        float2 e[8], o[8];
        e[0] = v[0]; o[0] = v[0];
        e[1] = v[1]; o[1] = twid<16, 1>(v[1]);
        e[2] = v[2]; o[2] = twid<16, 2>(v[2]);
        e[3] = v[3]; o[3] = twid<16, 3>(v[3]);
        e[4] = v[4]; o[4] = twid<16, 4>(v[4]);
        e[5] = v[5]; o[5] = twid<16, 5>(v[5]);
        e[6] = v[6]; o[6] = twid<16, 6>(v[6]);
        e[7] = v[7]; o[7] = twid<16, 7>(v[7]);
        Dft<8, PK>::run(e);
        Dft<8, PK>::run(o);
#pragma unroll
        for (int m = 0; m < 8; ++m) { v[2 * m] = e[m]; v[2 * m + 1] = o[m]; }
    }
};

}  // namespace b2d_fft
