// HBM-bound byte/element kernels of the quantized-linear path:
//   unpack             -- replaces optimum/quanto/library/extensions/cuda/unpack.cu:33-97 (1 byte/thread)
//   quantize_symmetric -- replaces the 3-4 ATen launches of optimum/quanto/library/quantize.py:51-55
//   dequantize_qbits   -- QBitsDequantizer.forward, optimum/quanto/tensor/qbits.py:27-49, as ONE launch
// All are 128-bit vectorised, grid-stride, launched on the caller's stream.
#include "../../include/quanto_b200.h"

#include "host_common.cuh"
#include "quantize_math.cuh"

namespace qb {

constexpr int kEwThreads = 256;
constexpr int kEwCtasPerSm = 16;  // 16 resident CTAs of 256 threads cover 2048 thr/SM x2 waves

// ---------------------------------------------------------------------------------------------
// unpack: out[p * n + i] = (in[i] >> (bits * p)) & mask        (planes concatenated along dim 0)
// ---------------------------------------------------------------------------------------------
template <int BITS>
__global__ void __launch_bounds__(kEwThreads) unpack_vec_kernel(const uint4* __restrict__ in, uint4* __restrict__ out,
                                                                int64_t n_vec) {
  constexpr int PLANES = 8 / BITS;
  constexpr uint32_t MASK = (BITS == 4) ? 0x0F0F0F0Fu : 0x03030303u;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_vec; i += stride) {
    const uint4 v = __ldcs(in + i);
#pragma unroll
    for (int p = 0; p < PLANES; ++p) {
      uint4 o;
      o.x = (v.x >> (BITS * p)) & MASK;
      o.y = (v.y >> (BITS * p)) & MASK;
      o.z = (v.z >> (BITS * p)) & MASK;
      o.w = (v.w >> (BITS * p)) & MASK;
      __stcs(out + static_cast<int64_t>(p) * n_vec + i, o);
    }
  }
}

template <int BITS>
__global__ void __launch_bounds__(kEwThreads) unpack_scalar_kernel(const uint8_t* __restrict__ in,
                                                                   uint8_t* __restrict__ out, int64_t n) {
  constexpr int PLANES = 8 / BITS;
  constexpr uint32_t MASK = (1u << BITS) - 1u;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint32_t v = in[i];
#pragma unroll
    for (int p = 0; p < PLANES; ++p) out[static_cast<int64_t>(p) * n + i] = static_cast<uint8_t>((v >> (BITS * p)) & MASK);
  }
}

// ---------------------------------------------------------------------------------------------
// quantize_symmetric
//   t = round_to_T(float(base) / float(scale))      -- the quotient is rounded to the INPUT dtype first
//   int8 : clamp(rint(t), -128, 127)                   (rint = half-to-even, as torch.round)
//   fp8  : clamp(t, -max, max) then RNE cast
// axis_mode: 0 per-tensor (scale[0]); 1 scale[outer index]; 2 scale[inner index]
// ---------------------------------------------------------------------------------------------
// UNR independent 16/32-byte loads are issued before any arithmetic so that every thread keeps UNR x 16 B (bf16/fp16)
// in flight: with one load per thread the kernel was latency-bound at 0.40 of the HBM roofline (round-1 measurement).
template <typename T, int OUT_DT, int VEC, int UNR>
__global__ void __launch_bounds__(kEwThreads)
    quantize_symmetric_kernel(const T* __restrict__ base, const T* __restrict__ scale, uint8_t* __restrict__ out,
                              int64_t numel, int64_t inner, int axis_mode) {
  const int64_t n_items = (numel + VEC - 1) / VEC;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  const float s0 = (axis_mode == 0) ? to_float<T>(scale[0]) : 1.f;
  const bool rcp0 = (axis_mode == 0) && rcp_is_safe<T>(s0);
  const float r0 = rcp0 ? __frcp_rn(s0) : 0.f;
  for (int64_t it0 = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; it0 < n_items; it0 += stride * UNR) {
    alignas(16) T v[UNR][VEC];
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      const int64_t it = it0 + u * stride;
      if (it < n_items) {
        const int64_t e0 = it * VEC;
        if constexpr (VEC > 1) {
          // VEC elements are contiguous, aligned, and (host guarantees inner % VEC == 0) inside one row
          if constexpr (sizeof(T) * VEC == 32) {
            *reinterpret_cast<uint4*>(&v[u][0]) = __ldcs(reinterpret_cast<const uint4*>(base + e0));
            *reinterpret_cast<uint4*>(&v[u][VEC / 2]) = __ldcs(reinterpret_cast<const uint4*>(base + e0) + 1);
          } else {
            *reinterpret_cast<uint4*>(&v[u][0]) = __ldcs(reinterpret_cast<const uint4*>(base + e0));
          }
        } else {
          v[u][0] = base[e0];
        }
      }
    }
#pragma unroll
    for (int u = 0; u < UNR; ++u) {
      const int64_t it = it0 + u * stride;
      if (it < n_items) {
        const int64_t e0 = it * VEC;
        alignas(8) uint8_t q[VEC];
        float s_row = s0, r_row = r0;
        bool use_rcp = rcp0;
        if (axis_mode == 1) {
          s_row = to_float<T>(scale[e0 / inner]);
          use_rcp = rcp_is_safe<T>(s_row);
          r_row = use_rcp ? __frcp_rn(s_row) : 0.f;
        }
        const int64_t col0 = (axis_mode == 2) ? (e0 % inner) : 0;
        // one loop per way of forming the quotient: a mode test inside the element loop cost ~10 extra instructions
        // per element (ncu: 21 executed per element, issue-bound at 0.38 of the HBM roofline)
        float t[VEC];
        if (axis_mode == 2) {
#pragma unroll
          for (int j = 0; j < VEC; ++j) t[j] = __fdiv_rn(to_float<T>(v[u][j]), to_float<T>(scale[col0 + j]));
        } else if (use_rcp) {
#pragma unroll
          for (int j = 0; j < VEC; ++j) t[j] = __fmul_rn(to_float<T>(v[u][j]), r_row);
        } else {
#pragma unroll
          for (int j = 0; j < VEC; ++j) t[j] = __fdiv_rn(to_float<T>(v[u][j]), s_row);
        }
        if constexpr (VEC % 2 == 0) {
#pragma unroll
          for (int j = 0; j < VEC; j += 2) rnd_pair<T>(t[j], t[j + 1]);
        } else {
          t[0] = rnd<T>(t[0]);
        }
#pragma unroll
        for (int j = 0; j < VEC; ++j) q[j] = quantize_one<OUT_DT>(t[j]);
        if constexpr (VEC == 8) {
          __stcs(reinterpret_cast<uint2*>(out + e0), *reinterpret_cast<uint2*>(q));
        } else {
          out[e0] = q[0];
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// dequantize_qbits (axis 0): canonical storage is `packed[Rp, G]` with plane p of byte (r, c) holding
// grouped row r + p*Rp (tensor/packed.py:45-69); grouped row R = n*(K/G)+g, and the axis-0 ungroup is a
// reshape (tensor/grouped.py:42-44), so plane p of byte i lands at flat output index i + p*Rp*G.
//   float shift: d = rnd(rnd(scale*q) - shift)      int shift: d = rnd(scale * (q - zp))
// ---------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ T dequant_one(uint32_t q, float s, float z, int zp, bool shift_is_int) {
  if (shift_is_int) {
    return from_float<T>(__fmul_rn(s, static_cast<float>(static_cast<int>(q) - zp)));
  }
  const float d1 = to_float<T>(from_float<T>(__fmul_rn(s, static_cast<float>(q))));
  return from_float<T>(__fsub_rn(d1, z));
}

template <typename T, int BITS>
__global__ void __launch_bounds__(kEwThreads)
    dequantize_qbits_kernel(const uint8_t* __restrict__ packed, const T* __restrict__ scale,
                            const void* __restrict__ shift, T* __restrict__ out, int64_t rows, int64_t packed_rows,
                            int group, int shift_is_int) {
  constexpr int PLANES = 8 / BITS;
  constexpr uint32_t MASK = (1u << BITS) - 1u;
  const int64_t n_bytes = packed_rows * group;
  const int64_t plane_elems = packed_rows * group;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  // 4 bytes per thread-iteration (group % 4 == 0 is guaranteed by the host)
  for (int64_t i4 = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i4 * 4 < n_bytes; i4 += stride) {
    const int64_t i = i4 * 4;
    const uint32_t w = __ldcs(reinterpret_cast<const uint32_t*>(packed + i));
    const int64_t r = i / group;
#pragma unroll
    for (int p = 0; p < PLANES; ++p) {
      const int64_t row = r + static_cast<int64_t>(p) * packed_rows;
      if (row >= rows) continue;
      const float s = to_float<T>(scale[row]);
      float z = 0.f;
      int zp = 0;
      if (shift_is_int) zp = static_cast<int>(static_cast<int8_t>(static_cast<const uint8_t*>(shift)[row]));
      else z = to_float<T>(static_cast<const T*>(shift)[row]);
      alignas(16) T o[4];
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const uint32_t q = (w >> (8 * b + BITS * p)) & MASK;
        o[b] = dequant_one<T>(q, s, z, zp, shift_is_int != 0);
      }
      T* dst = out + i + static_cast<int64_t>(p) * plane_elems;
      if constexpr (sizeof(T) == 2) {
        *reinterpret_cast<uint2*>(dst) = *reinterpret_cast<uint2*>(o);
      } else {
        *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<uint4*>(o);
      }
    }
  }
}

}  // namespace qb

using namespace qb;

extern "C" {

int qb200_unpack(const uint8_t* in, uint8_t* out, int64_t n_bytes, int bits, void* stream) {
  if (bits != 2 && bits != 4) return fail(ERR_ARG, "unpack: bits must be 2 or 4, got %d", bits);
  if (n_bytes < 0 || (n_bytes > 0 && (in == nullptr || out == nullptr))) return fail(ERR_ARG, "unpack: bad buffer");
  if (n_bytes == 0) return OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool vec = n_bytes % 16 == 0 && aligned16(in) && aligned16(out);
  return dispatch_bits(bits, [&](auto BITS) {
    if (vec)
      unpack_vec_kernel<BITS><<<capped_grid(n_bytes / 16, kEwThreads, kEwCtasPerSm), kEwThreads, 0, st>>>(
          reinterpret_cast<const uint4*>(in), reinterpret_cast<uint4*>(out), n_bytes / 16);
    else
      unpack_scalar_kernel<BITS><<<capped_grid(n_bytes, kEwThreads, kEwCtasPerSm), kEwThreads, 0, st>>>(in, out, n_bytes);
    return check_cuda(cudaGetLastError(), "unpack launch");
  });
}

int qb200_quantize_symmetric(const void* base, const void* scale, void* out, int64_t outer, int64_t inner,
                             int axis_mode, int in_dtype, int out_dtype, void* stream) {
  if (!is_float_dtype(in_dtype)) return fail(ERR_ARG, "quantize_symmetric: input dtype %d not floating point", in_dtype);
  if (!is_code_dtype(out_dtype)) return fail(ERR_ARG, "quantize_symmetric: unsupported target dtype %d", out_dtype);
  if (axis_mode < 0 || axis_mode > 2) return fail(ERR_ARG, "quantize_symmetric: axis_mode %d", axis_mode);
  if (outer < 0 || inner < 0)
    return fail(ERR_ARG, "quantize_symmetric: negative shape (%lld x %lld)", (long long)outer, (long long)inner);
  const int64_t numel = outer * inner;
  if (numel == 0) return OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool vec = inner % 8 == 0 && numel % 8 == 0 && aligned16(base) && reinterpret_cast<uintptr_t>(out) % 8 == 0;
  return dispatch_float(in_dtype, [&](auto in) {
    return dispatch_code8(out_dtype, [&](auto OUT) {
      using T = typename decltype(in)::T;
      const T* b = static_cast<const T*>(base);
      const T* s = static_cast<const T*>(scale);
      uint8_t* o = static_cast<uint8_t*>(out);
      if (vec) {
        constexpr int UNR = 4;
        quantize_symmetric_kernel<T, OUT, 8, UNR>
            <<<capped_grid((numel / 8 + UNR - 1) / UNR, kEwThreads, kEwCtasPerSm), kEwThreads, 0, st>>>(
                b, s, o, numel, inner, axis_mode);
      } else {
        quantize_symmetric_kernel<T, OUT, 1, 1><<<capped_grid(numel, kEwThreads, kEwCtasPerSm), kEwThreads, 0, st>>>(
            b, s, o, numel, inner, axis_mode);
      }
      return check_cuda(cudaGetLastError(), "quantize_symmetric launch");
    });
  });
}

int qb200_dequantize_qbits(const uint8_t* packed, const void* scale, const void* shift, void* out, int64_t n,
                           int64_t k, int group, int bits, int dtype, int shift_is_int, void* stream) {
  if (bits != 2 && bits != 4) return fail(ERR_ARG, "dequantize_qbits: bits must be 2 or 4, got %d", bits);
  if (n <= 0 || k <= 0 || group <= 0 || (n * k) % group != 0 || group % 4 != 0)
    return fail(ERR_ARG, "dequantize_qbits: bad shape (N=%lld K=%lld group=%d)", (long long)n, (long long)k, group);
  if (reinterpret_cast<uintptr_t>(packed) % 4 != 0 || !aligned16(out))
    return fail(ERR_ARG, "dequantize_qbits: packed must be 4-byte and out 16-byte aligned");
  if (!is_float_dtype(dtype)) return fail(ERR_ARG, "dequantize_qbits: dtype %d not floating point", dtype);
  const int64_t rows = n * k / group;
  const int planes = 8 / bits;
  const int64_t packed_rows = (rows + planes - 1) / planes;
  const int grid = capped_grid(packed_rows * group / 4, kEwThreads, kEwCtasPerSm);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return dispatch_float(dtype, [&](auto dt) {
    return dispatch_bits(bits, [&](auto BITS) {
      using T = typename decltype(dt)::T;
      dequantize_qbits_kernel<T, BITS><<<grid, kEwThreads, 0, st>>>(
          packed, static_cast<const T*>(scale), shift, static_cast<T*>(out), rows, packed_rows, group, shift_is_int);
      return check_cuda(cudaGetLastError(), "dequantize_qbits launch");
    });
  });
}

}  // extern "C"
