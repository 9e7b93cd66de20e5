// HBM-bound byte/element kernels of the quantized-linear path:
//   unpack             -- replaces optimum/quanto/library/extensions/cuda/unpack.cu:33-97 (1 byte/thread)
//   quantize_symmetric -- replaces the 3-4 ATen launches of optimum/quanto/library/quantize.py:51-55
//   dequantize_qbits   -- QBitsDequantizer.forward, optimum/quanto/tensor/qbits.py:27-49, as ONE launch
// All are 128-bit vectorised, grid-stride, launched on the caller's stream.
#include <type_traits>

#include "common.cuh"
#include "quantize_math.cuh"

namespace qb {

constexpr int kEwThreads = 256;

static inline int ew_grid(int64_t work_items) {
  int64_t blocks = (work_items + kEwThreads - 1) / kEwThreads;
  int64_t cap = static_cast<int64_t>(kNumSMsH100) * 16;  // 16 resident CTAs of 256 threads cover 2048 thr/SM x2 waves
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

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

int launch_unpack(const uint8_t* in, uint8_t* out, int64_t n_bytes, int bits, cudaStream_t stream) {
  if (bits != 2 && bits != 4) return ERR_ARG;
  if (n_bytes < 0) return ERR_ARG;
  if (n_bytes == 0) return OK;
  const bool vec = (n_bytes % 16 == 0) && (reinterpret_cast<uintptr_t>(in) % 16 == 0) &&
                   (reinterpret_cast<uintptr_t>(out) % 16 == 0);
  if (vec) {
    const int64_t n_vec = n_bytes / 16;
    const int grid = ew_grid(n_vec);
    if (bits == 4)
      unpack_vec_kernel<4><<<grid, kEwThreads, 0, stream>>>(reinterpret_cast<const uint4*>(in),
                                                            reinterpret_cast<uint4*>(out), n_vec);
    else
      unpack_vec_kernel<2><<<grid, kEwThreads, 0, stream>>>(reinterpret_cast<const uint4*>(in),
                                                            reinterpret_cast<uint4*>(out), n_vec);
  } else {
    const int grid = ew_grid(n_bytes);
    if (bits == 4)
      unpack_scalar_kernel<4><<<grid, kEwThreads, 0, stream>>>(in, out, n_bytes);
    else
      unpack_scalar_kernel<2><<<grid, kEwThreads, 0, stream>>>(in, out, n_bytes);
  }
  return cudaGetLastError() == cudaSuccess ? OK : ERR_CUDA;
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

template <typename T, int OUT_DT>
static int launch_qs_t(const void* base, const void* scale, void* out, int64_t numel, int64_t inner, int axis_mode,
                       cudaStream_t stream) {
  const bool vec = (inner % 8 == 0) && (numel % 8 == 0) && (reinterpret_cast<uintptr_t>(base) % 16 == 0) &&
                   (reinterpret_cast<uintptr_t>(out) % 8 == 0);
  if (vec) {
    constexpr int UNR = 4;
    const int grid = ew_grid((numel / 8 + UNR - 1) / UNR);
    quantize_symmetric_kernel<T, OUT_DT, 8, UNR><<<grid, kEwThreads, 0, stream>>>(
        static_cast<const T*>(base), static_cast<const T*>(scale), static_cast<uint8_t*>(out), numel, inner, axis_mode);
  } else {
    const int grid = ew_grid(numel);
    quantize_symmetric_kernel<T, OUT_DT, 1, 1><<<grid, kEwThreads, 0, stream>>>(
        static_cast<const T*>(base), static_cast<const T*>(scale), static_cast<uint8_t*>(out), numel, inner, axis_mode);
  }
  return cudaGetLastError() == cudaSuccess ? OK : ERR_CUDA;
}

template <typename T>
static int launch_qs_o(const void* base, const void* scale, void* out, int64_t numel, int64_t inner, int axis_mode,
                       int out_dt, cudaStream_t stream) {
  switch (out_dt) {
    case DT_I8: return launch_qs_t<T, DT_I8>(base, scale, out, numel, inner, axis_mode, stream);
    case DT_E4M3: return launch_qs_t<T, DT_E4M3>(base, scale, out, numel, inner, axis_mode, stream);
    case DT_E5M2: return launch_qs_t<T, DT_E5M2>(base, scale, out, numel, inner, axis_mode, stream);
    case DT_E4M3FNUZ: return launch_qs_t<T, DT_E4M3FNUZ>(base, scale, out, numel, inner, axis_mode, stream);
    default: return ERR_ARG;
  }
}

int launch_quantize_symmetric(const void* base, const void* scale, void* out, int64_t outer, int64_t inner,
                              int axis_mode, int in_dt, int out_dt, cudaStream_t stream) {
  if (outer < 0 || inner < 0 || axis_mode < 0 || axis_mode > 2) return ERR_ARG;
  const int64_t numel = outer * inner;
  if (numel == 0) return OK;
  switch (in_dt) {
    case DT_F32: return launch_qs_o<float>(base, scale, out, numel, inner, axis_mode, out_dt, stream);
    case DT_F16: return launch_qs_o<__half>(base, scale, out, numel, inner, axis_mode, out_dt, stream);
    case DT_BF16: return launch_qs_o<__nv_bfloat16>(base, scale, out, numel, inner, axis_mode, out_dt, stream);
    default: return ERR_ARG;
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

template <typename T>
static int launch_deq_t(const uint8_t* packed, const void* scale, const void* shift, void* out, int64_t rows,
                        int64_t packed_rows, int group, int bits, int shift_is_int, cudaStream_t stream) {
  const int grid = ew_grid(packed_rows * group / 4);
  if (bits == 4)
    dequantize_qbits_kernel<T, 4><<<grid, kEwThreads, 0, stream>>>(packed, static_cast<const T*>(scale), shift,
                                                                   static_cast<T*>(out), rows, packed_rows, group,
                                                                   shift_is_int);
  else
    dequantize_qbits_kernel<T, 2><<<grid, kEwThreads, 0, stream>>>(packed, static_cast<const T*>(scale), shift,
                                                                   static_cast<T*>(out), rows, packed_rows, group,
                                                                   shift_is_int);
  return cudaGetLastError() == cudaSuccess ? OK : ERR_CUDA;
}

int launch_dequantize_qbits(const uint8_t* packed, const void* scale, const void* shift, void* out, int64_t n,
                            int64_t k, int group, int bits, int dt, int shift_is_int, cudaStream_t stream) {
  if ((bits != 2 && bits != 4) || n <= 0 || k <= 0 || group <= 0) return ERR_ARG;
  if ((n * k) % group != 0 || group % 4 != 0) return ERR_ARG;
  if (reinterpret_cast<uintptr_t>(packed) % 4 != 0 || reinterpret_cast<uintptr_t>(out) % 16 != 0) return ERR_ARG;
  const int64_t rows = n * k / group;
  const int planes = 8 / bits;
  const int64_t packed_rows = (rows + planes - 1) / planes;
  switch (dt) {
    case DT_F32: return launch_deq_t<float>(packed, scale, shift, out, rows, packed_rows, group, bits, shift_is_int, stream);
    case DT_F16: return launch_deq_t<__half>(packed, scale, shift, out, rows, packed_rows, group, bits, shift_is_int, stream);
    case DT_BF16:
      return launch_deq_t<__nv_bfloat16>(packed, scale, shift, out, rows, packed_rows, group, bits, shift_is_int, stream);
    default: return ERR_ARG;
  }
}

}  // namespace qb
