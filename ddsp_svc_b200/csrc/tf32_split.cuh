// fp32 -> (tf32 hi, tf32 lo) split for 3xTF32 library GEMMs: x = hi + lo + O(2^-22 |x|), both parts exactly
// representable in TF32 (10-bit mantissa, round to nearest even on the dropped 13 bits).  Shared by b2d_split_tf32
// (unit2control.cu) and, through tf32_emit, the kernels that write a GEMM operand directly (reflow*.cu, diffusion*.cu).
// A NaN becomes the TF32 quiet NaN 0x7FFFE000: the rounding add would carry the low payload bits of a NaN into the
// exponent and sign (the canonical NaN 0x7FFFFFFF that device arithmetic produces came out as -0).  +-inf split into
// (+-inf, +0).  Finite values above the largest TF32 value round to hi = +-inf, lo = -+inf.
#pragma once

__device__ __forceinline__ float tf32_rn(float x) {
    uint32_t u = __float_as_uint(x);
    if ((u & 0x7FFFFFFFu) > 0x7F800000u) return __uint_as_float(0x7FFFE000u);
    u += 0x00000FFFu + ((u >> 13) & 1u);
    return __uint_as_float(u & 0xFFFFE000u);
}
__device__ __forceinline__ void tf32_split(float v, float& h, float& l) {
    h = tf32_rn(v);
    l = tf32_rn(v == h ? 0.f : v - h);              // v == h also for +-inf, where v - h would be NaN
}

// element i of a GEMM operand: the TF32 (hi, lo) halves of a 3xTF32 product, or v itself into hi when lo is NULL (fp32)
__device__ __forceinline__ void tf32_emit(float v, float* __restrict__ hi, float* __restrict__ lo, size_t i) {
    if (lo) {
        float h, l;
        tf32_split(v, h, l);
        hi[i] = h;
        lo[i] = l;
    } else {
        hi[i] = v;
    }
}
// tf32_emit for an optional operand: nothing when hi is NULL
__device__ __forceinline__ void tf32_emit_opt(float v, float* __restrict__ hi, float* __restrict__ lo, size_t i) {
    if (hi) tf32_emit(v, hi, lo, i);
}
