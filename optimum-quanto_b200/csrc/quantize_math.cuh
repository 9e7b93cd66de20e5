// Exact (bit-for-bit with the reference's CPU arithmetic) scalar building blocks shared by the quantisation kernels
// of elementwise.cu and freeze.cu.  Every step uses the *_rn intrinsics so that ptxas cannot contract an add/mul
// pair into an fma or replace a division by a reciprocal multiply.
#pragma once

#include <type_traits>

#include "common.cuh"

namespace qb {

// round a float to T (nearest even) and widen it again: the value an ATen op on dtype T hands to the next op
template <typename T>
__device__ __forceinline__ float rnd(float v) {
  return to_float<T>(from_float<T>(v));
}

// rnd<T> of two values at once: one packed F2FP conversion instead of two scalar ones for the 16-bit types
template <typename T>
__device__ __forceinline__ void rnd_pair(float& a, float& b) {
  if constexpr (std::is_same<T, __nv_bfloat16>::value) {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    a = __low2float(h);
    b = __high2float(h);
  } else if constexpr (std::is_same<T, __half>::value) {
    const __half2 h = __floats2half2_rn(a, b);
    a = __low2float(h);
    b = __high2float(h);
  }
}

// For bf16 operands the quotient rounded to bf16 can be obtained from a * rcp_rn(s) instead of an IEEE division
// (a tenth of the instructions): the fp32 error of a*rcp(s) is <= 2^-22 relative, while a/s for 8-bit significands
// stays >= 2^-17 (relative) away from every bf16 rounding boundary unless it lies exactly on a representable value --
// exact ties cannot occur (an odd 9-bit midpoint times an 8-bit significand never fits in 8 bits).  So
// rnd_bf16(a * rcp(s)) == rnd_bf16(a / s) bit for bit for normal quotients; a subnormal quotient is < 2^-126 either
// way and quantises to 0 (int8 / int4 / fp8) whatever its last bits.  Guarded to scales whose reciprocal is a normal
// number.  fp16 (11-bit significands: margin 2^-23) and fp32 keep the exact division.
template <typename T>
__device__ __forceinline__ bool rcp_is_safe(float s) {
  const float a = fabsf(s);
  return std::is_same<T, __nv_bfloat16>::value && a > 1e-30f && a < 1e30f;
}

// Round-half-even of a float already clamped to |t| <= 2^22, as the integer's two's-complement bits: at 1.5 * 2^23 the
// fp32 ulp is 1, so the RN addition rounds t to an integer (ties to the even mantissa = the even integer) and the sum's
// bit pattern is 0x4B400000 + n.  Clamping before rounding equals clamping after it because the bounds are integers.
__device__ __forceinline__ int rint_bits(float t_clamped) {
  return __float_as_int(__fadd_rn(t_clamped, 12582912.f)) - 0x4B400000;
}

// clamp + cast of quantize_symmetric (optimum/quanto/library/quantize.py:51-55); t is already rounded to the input dtype
template <int OUT_DT>
__device__ __forceinline__ uint8_t quantize_one(float t) {
  if constexpr (OUT_DT == DT_I8) {
    // NaN -> 0 (what the reference's NaN -> int8 cast gives on x86 and on CUDA: an all-zero row has scale 0 and
    // quotient 0/0), clamp, then round-half-even through the 1.5 * 2^23 addition (see rint_bits): FMA/ALU pipes only.
    // F2I / FRND / F2F run on the quarter-rate XU pipe, which bounded the first version of these kernels (ncu: XU 46-74 %).
    float c = (t != t) ? 0.f : t;
    c = fminf(fmaxf(c, -128.f), 127.f);
    return static_cast<uint8_t>(rint_bits(c) & 0xFF);
  } else if constexpr (OUT_DT == DT_E4M3) {
    if (t != t) return static_cast<uint8_t>(0x7Fu | ((__float_as_uint(t) >> 24) & 0x80u));  // NaN stays NaN (torch)
    float c = fminf(fmaxf(t, -448.f), 448.f);
    return static_cast<uint8_t>(__nv_cvt_float_to_fp8(c, __NV_SATFINITE, __NV_E4M3));
  } else if constexpr (OUT_DT == DT_E4M3FNUZ) {
    // float8_e4m3fnuz (optimum/quanto/tensor/qtype.py:63): no native convert.  Round-half-even to 3 mantissa
    // bits on the fp32 pattern (normals) / to a multiple of 2^-10 (subnormals); zero has no sign, NaN is 0x80.
    if (t != t) return 0x80u;
    const float c = fminf(fmaxf(t, -240.f), 240.f);
    const float a = fabsf(c);
    uint32_t b;
    if (a < 0.0078125f) {
      b = static_cast<uint32_t>(rint_bits(a * 1024.f));  // 0..8 (8 = the smallest normal)
    } else {
      uint32_t u = __float_as_uint(a);
      u += 0x7FFFFu + ((u >> 20) & 1u);
      b = ((((u >> 23) & 0xFFu) - 119u) << 3) | ((u >> 20) & 7u);
    }
    return static_cast<uint8_t>(b == 0u ? 0u : (b | (c < 0.f ? 0x80u : 0u)));
  } else {
    if (t != t) return static_cast<uint8_t>(0x7Fu | ((__float_as_uint(t) >> 24) & 0x80u));
    float c = fminf(fmaxf(t, -57344.f), 57344.f);
    return static_cast<uint8_t>(__nv_cvt_float_to_fp8(c, __NV_SATFINITE, __NV_E5M2));
  }
}

// the payload of an 8-bit code of dtype Q (the low byte of v) as a float: the int8 value or the fp8 value
template <int Q>
__device__ __forceinline__ float decode8(uint32_t v) {
  if constexpr (Q == DT_I8) return static_cast<float>(static_cast<int8_t>(static_cast<uint8_t>(v)));
  else if constexpr (Q == DT_E4M3) return e4m3_to_float(static_cast<uint8_t>(v));
  else if constexpr (Q == DT_E5M2) return e5m2_to_float(static_cast<uint8_t>(v));
  else return e4m3fnuz_to_float(static_cast<uint8_t>(v));
}

// quanto::quantize_affine for one element (optimum/quanto/library/quantize.py:71-78), arithmetic in dtype T:
//   float shift : clamp(rint(rnd(rnd(b + z) / s)), 0, qmax)
//   zero-point  : clamp(rnd(rint(rnd(b / s)) + zp), 0, qmax)
// NaN (0/0 of a constant group) maps to 0, what the reference's NaN -> uint8 cast yields on x86.
template <typename T, bool ZP>
__device__ __forceinline__ uint32_t affine_quantize_one(float b, float s, float z, float qmax) {
  float r;
  if constexpr (ZP) r = rnd<T>(__fadd_rn(rintf(rnd<T>(__fdiv_rn(b, s))), z));
  else r = rintf(rnd<T>(__fdiv_rn(rnd<T>(__fadd_rn(b, z)), s)));
  r = fminf(fmaxf(r, 0.f), qmax);  // fmaxf returns the non-NaN operand
  return static_cast<uint32_t>(r);
}

// The same for 8 elements of one group, rounding through rint_bits (no XU-pipe conversions) and, when
// FAST (bf16 with a normal reciprocal, see rcp_is_safe), the division as a multiplication by r = rcp_rn(s).
// Zero-point form: rnd(rint(t) + zp) == rint(t) + zp whenever the sum can survive the clamp (integers up to 256 are
// exact in every T), so the zero-point is added as an integer after a pre-clamp that rules out overflow.
template <typename T, bool ZP, bool FAST>
__device__ __forceinline__ void affine_quantize8(const float (&f)[8], float s, float r, float z, int qmax,
                                                 int shift_left, uint32_t (&bytes)[8]) {
  float t[8];
#pragma unroll
  for (int j = 0; j < 8; j += 2) {
    float a = f[j], b = f[j + 1];
    if constexpr (!ZP) {
      a = __fadd_rn(a, z);
      b = __fadd_rn(b, z);
      rnd_pair<T>(a, b);
    }
    if constexpr (FAST) {
      a = __fmul_rn(a, r);
      b = __fmul_rn(b, r);
    } else {
      a = __fdiv_rn(a, s);
      b = __fdiv_rn(b, s);
    }
    rnd_pair<T>(a, b);
    t[j] = a;
    t[j + 1] = b;
  }
  const int zp = ZP ? static_cast<int>(z) : 0;
  const float qmaxf = static_cast<float>(qmax);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    int v;
    if constexpr (ZP) {
      // NaN -> -65536 (fmaxf returns the non-NaN operand): NaN + zp stays NaN in the reference and casts to 0
      v = rint_bits(fminf(fmaxf(t[j], -65536.f), 65536.f)) + zp;
      v = max(0, min(qmax, v));
    } else {
      v = rint_bits(fminf(fmaxf(t[j], 0.f), qmaxf));  // NaN -> 0
    }
    bytes[j] |= static_cast<uint32_t>(v) << shift_left;
  }
}

// 8 consecutive elements of T (16-byte aligned address) widened to float, streaming load
template <typename T>
__device__ __forceinline__ void load8_stream(const T* __restrict__ p, float (&f)[8]) {
  if constexpr (sizeof(T) == 2) {
    const uint4 r = __ldcs(reinterpret_cast<const uint4*>(p));
    const T* e = reinterpret_cast<const T*>(&r);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = to_float<T>(e[j]);
  } else {
    const uint4 a = __ldcs(reinterpret_cast<const uint4*>(p));
    const uint4 b = __ldcs(reinterpret_cast<const uint4*>(p) + 1);
    f[0] = __uint_as_float(a.x); f[1] = __uint_as_float(a.y); f[2] = __uint_as_float(a.z); f[3] = __uint_as_float(a.w);
    f[4] = __uint_as_float(b.x); f[5] = __uint_as_float(b.y); f[6] = __uint_as_float(b.z); f[7] = __uint_as_float(b.w);
  }
}

}  // namespace qb
