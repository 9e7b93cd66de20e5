// Shape-agnostic qbytes_mm on CUDA cores.  This is the path for configurations the tensor-core kernels do not
// take (K not a multiple of 16 bytes, fp32 activations, exotic dtype mixes).  It follows the reference's rounding
// order literally (optimum/quanto/library/qbytes_mm.py:25-50):
//   int8 x int8 : acc = int32 sum ; out = rnd_T(fp32(acc) * fp32(scale[n]))
//   otherwise   : A' = rnd_T(A) ; Ws = rnd_T(scale[n] * W) ; out = rnd_T(sum_k A'*Ws)  (fp32 accumulate)
#include "host_common.cuh"

namespace qb {

constexpr int ST = 64;   // tile edge
constexpr int SK = 16;   // k step

__device__ __forceinline__ float load_as_float(const void* p, int dt, size_t idx) {
  switch (dt) {
    case DT_F32: return static_cast<const float*>(p)[idx];
    case DT_F16: return __half2float(static_cast<const __half*>(p)[idx]);
    case DT_BF16: return __bfloat162float(static_cast<const __nv_bfloat16*>(p)[idx]);
    case DT_I8: return static_cast<float>(static_cast<const int8_t*>(p)[idx]);
    case DT_U8: return static_cast<float>(static_cast<const uint8_t*>(p)[idx]);
    case DT_E4M3: return e4m3_to_float(static_cast<const uint8_t*>(p)[idx]);
    case DT_E4M3FNUZ: return e4m3fnuz_to_float(static_cast<const uint8_t*>(p)[idx]);
    default: return e5m2_to_float(static_cast<const uint8_t*>(p)[idx]);
  }
}

template <typename T, bool INT_PATH>
__global__ void __launch_bounds__(256)
    qbytes_mm_simt_kernel(const void* __restrict__ A, const void* __restrict__ W, const T* __restrict__ scales,
                          const T* __restrict__ bias, T* __restrict__ out, int M, int N, int K, int a_dt, int w_dt) {
  __shared__ float sa[SK][ST + 1];
  __shared__ float sw[SK][ST + 1];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int m0 = blockIdx.y * ST, n0 = blockIdx.x * ST;
  float accf[4][4];
  int acci[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) { accf[i][j] = 0.f; acci[i][j] = 0; }

  for (int k0 = 0; k0 < K; k0 += SK) {
    for (int e = threadIdx.x; e < ST * SK; e += 256) {
      const int r = e / SK, kk = e % SK;
      const int k = k0 + kk;
      float av = 0.f, wv = 0.f;
      if (k < K) {
        if (m0 + r < M) {
          av = load_as_float(A, a_dt, static_cast<size_t>(m0 + r) * K + k);
          if (!INT_PATH) av = to_float<T>(from_float<T>(av));  // activations.to(scales.dtype)
        }
        if (n0 + r < N) {
          wv = load_as_float(W, w_dt, static_cast<size_t>(n0 + r) * K + k);
          if (!INT_PATH) wv = to_float<T>(from_float<T>(__fmul_rn(to_float<T>(scales[n0 + r]), wv)));
        }
      }
      sa[kk][r] = av;
      sw[kk][r] = wv;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < SK; ++kk) {
      float a[4], w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = sa[kk][ty * 4 + i]; w[i] = sw[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (INT_PATH) acci[i][j] += static_cast<int>(a[i]) * static_cast<int>(w[j]);
          else accf[i][j] = fmaf(a[i], w[j], accf[i][j]);
        }
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + j;
      if (m < M && n < N) {
        float f = INT_PATH ? __fmul_rn(__int2float_rn(acci[i][j]), to_float<T>(scales[n])) : accf[i][j];
        T r = from_float<T>(f);
        if (bias != nullptr) r = from_float<T>(__fadd_rn(to_float<T>(r), to_float<T>(bias[n])));
        out[static_cast<size_t>(m) * N + n] = r;
      }
    }
}

int launch_qbytes_mm_simt(const void* A, const void* W, const void* scales, const void* bias, void* out, int M, int N,
                          int K, int a_dt, int w_dt, int out_dt, cudaStream_t stream) {
  dim3 grid((N + ST - 1) / ST, (M + ST - 1) / ST);
  const bool int_path = a_dt == DT_I8 && w_dt == DT_I8;
  return dispatch_float(out_dt, [&](auto dt) {
    using T = typename decltype(dt)::T;
    auto launch = [&](auto INT_PATH) {
      qbytes_mm_simt_kernel<T, INT_PATH><<<grid, 256, 0, stream>>>(A, W, static_cast<const T*>(scales),
                                                                   static_cast<const T*>(bias), static_cast<T*>(out), M,
                                                                   N, K, a_dt, w_dt);
      return check_cuda(cudaGetLastError(), "qbytes_mm CUDA-core launch");
    };
    return int_path ? launch(std::true_type{}) : launch(std::false_type{});
  });
}

// ---------------------------------------------------------------------------------------------
// Shape-agnostic fused packed-int4 / int2 linear on CUDA cores: the native path for everything the tensor-core kernels
// of qb200_qbits_mm do not take (2-bit weights, odd N, K not a multiple of 16, group sizes other than 32 / 64k, fp32).
// Axis-0 canonical storage (tensor/packed.py:45-69, tensor/grouped.py:17-30): grouped row R = n * (K / G) + k / G lives
// in bit plane R / Rp of byte row R % Rp.  Operands are dequantised with the reference's rounding order
// (tensor/qbits.py:34-45), products accumulate in fp32, one rounding to T, bias added after it.
// ---------------------------------------------------------------------------------------------
template <typename T, int BITS>
__global__ void __launch_bounds__(256)
    qbits_mm_simt_kernel(const T* __restrict__ X, const uint8_t* __restrict__ packed, const T* __restrict__ scale,
                         const void* __restrict__ shift, const T* __restrict__ bias, T* __restrict__ out, int M, int N,
                         int K, int group, int64_t packed_rows, int shift_is_int, int64_t ld, int64_t col0) {
  constexpr uint32_t MASK = (1u << BITS) - 1u;
  __shared__ float sa[SK][ST + 1];
  __shared__ float sw[SK][ST + 1];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int m0 = blockIdx.y * ST, n0 = blockIdx.x * ST;
  const int gpr = K / group;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < K; k0 += SK) {
    for (int e = threadIdx.x; e < ST * SK; e += 256) {
      const int r = e / SK, kk = e % SK;
      const int k = k0 + kk;
      float av = 0.f, wv = 0.f;
      if (k < K) {
        if (m0 + r < M) av = to_float<T>(X[static_cast<size_t>(m0 + r) * K + k]);
        if (n0 + r < N) {
          const int64_t row = static_cast<int64_t>(n0 + r) * gpr + k / group;
          const int64_t plane = row / packed_rows, brow = row - plane * packed_rows;
          const uint32_t q = (static_cast<uint32_t>(packed[brow * group + (k % group)]) >> (BITS * plane)) & MASK;
          const float sc = to_float<T>(scale[row]);
          if (shift_is_int) {
            const int zp = static_cast<int>(static_cast<int8_t>(static_cast<const uint8_t*>(shift)[row]));
            wv = to_float<T>(from_float<T>(__fmul_rn(sc, static_cast<float>(static_cast<int>(q) - zp))));
          } else {
            const float d1 = to_float<T>(from_float<T>(__fmul_rn(sc, static_cast<float>(q))));
            wv = to_float<T>(from_float<T>(__fsub_rn(d1, to_float<T>(static_cast<const T*>(shift)[row]))));
          }
        }
      }
      sa[kk][r] = av;
      sw[kk][r] = wv;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < SK; ++kk) {
      float a[4], w[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = sa[kk][ty * 4 + i]; w[i] = sw[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], w[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + j;
      if (m < M && n < N) {
        T r = from_float<T>(acc[i][j]);
        if (bias != nullptr) r = from_float<T>(__fadd_rn(to_float<T>(r), to_float<T>(bias[n])));
        out[static_cast<size_t>(m) * ld + col0 + n] = r;
      }
    }
}

int launch_qbits_mm_simt(const void* x, const uint8_t* packed, const void* scale, const void* shift, const void* bias,
                         void* out, int M, int N, int K, int group, int bits, int dt, int shift_is_int, int64_t ld,
                         int64_t col0, cudaStream_t stream) {
  dim3 grid((N + ST - 1) / ST, (M + ST - 1) / ST);
  const int64_t rows = static_cast<int64_t>(N) * (K / group);
  const int planes = 8 / bits;
  const int64_t packed_rows = (rows + planes - 1) / planes;
  return dispatch_float(dt, [&](auto t) {
    return dispatch_bits(bits, [&](auto BITS) {
      using T = typename decltype(t)::T;
      qbits_mm_simt_kernel<T, BITS><<<grid, 256, 0, stream>>>(static_cast<const T*>(x), packed,
                                                              static_cast<const T*>(scale), shift,
                                                              static_cast<const T*>(bias), static_cast<T*>(out), M, N,
                                                              K, group, packed_rows, shift_is_int, ld, col0);
      return check_cuda(cudaGetLastError(), "qbits_mm CUDA-core launch");
    });
  });
}

}  // namespace qb
