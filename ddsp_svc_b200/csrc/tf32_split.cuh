// fp32 -> (tf32 hi, tf32 lo) split for 3xTF32 library GEMMs: x = hi + lo + O(2^-22 |x|), both parts exactly
// representable in TF32 (10-bit mantissa, round to nearest even on the dropped 13 bits).  Shared by b2d_split_tf32
// (unit2control.cu) and the kernels that emit a GEMM operand directly in split form (reflow.cu).
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
