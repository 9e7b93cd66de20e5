// The reference's QLayerNorm (optimum/quanto/nn/qlayernorm.py:27-53) as one launch:
//
//   F.layer_norm(input, normalized_shape, weight, bias, eps)      qlayernorm.py:52-53, after qfallback dequantizes an
//                                                                  ActivationQBytesTensor input (tensor/qbytes.py:23-31)
//   quantize_symmetric(y, qtype, None, output_scale)              the quantize_output hook (nn/qmodule.py:296-302 ->
//                                                                  library/quantize.py:51-55)
//
// per row of H elements:
//   x = the float input, or rnd_T(s_in * payload) for 8-bit codes (QBytesTensor.dequantize)
//   mean, then the biased variance of (x - mean), both summed in fp32; rstd = 1 / sqrt(var + eps) correctly rounded
//   y = rnd_T(gamma * (x - mean) * rstd + beta)       gamma, beta optional, in T
//   out = quantize_symmetric(y, out_scale)            quantize_math.cuh: quotient rounded to T, rint / clamp, cast
//       | y                                           (float output)
// The input is read from memory once for rows of up to kCacheVecs * 8 * kMaxThreads = 16384 elements: each thread keeps
// its share of the row in registers between the mean, the variance and the output pass.  Longer rows are read again by
// the variance and the output pass.  One warp per row while the row fits in the warp's registers (H <= 1024), one CTA
// per row above.
#include "../../include/quanto_b200.h"

#include "host_common.cuh"
#include "quantize_math.cuh"

namespace qb {

constexpr int kFloatIO = -1;      // template IN / OUT: floats in T instead of 8-bit codes
constexpr int kCacheVecs = 4;     // chunks of 8 elements each thread keeps in registers
constexpr int kWarpThreads = 256; // warp-per-row CTAs: 8 rows
constexpr int kMaxThreads = 512;  // CTA-per-row: up to 512 threads x 32 cached elements

// elements [e0, e0 + 8) of a row of H: a 16-byte vector (two for fp32, 8 bytes for codes) when `vec` (H % 8 == 0 and
// every buffer 16-byte aligned), else element by element with zeros past the end
template <typename T, int IN>
__device__ __forceinline__ void load_chunk(const void* __restrict__ row, int e0, int H, bool vec, float s_in,
                                           float (&f)[8]) {
  if constexpr (IN == kFloatIO) {
    const T* p = static_cast<const T*>(row) + e0;
    if (vec) {
      if constexpr (sizeof(T) == 2) {
        const uint4 r = *reinterpret_cast<const uint4*>(p);
        const T* e = reinterpret_cast<const T*>(&r);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = to_float<T>(e[j]);
      } else {
        const uint4 a = reinterpret_cast<const uint4*>(p)[0], b = reinterpret_cast<const uint4*>(p)[1];
        f[0] = __uint_as_float(a.x); f[1] = __uint_as_float(a.y); f[2] = __uint_as_float(a.z); f[3] = __uint_as_float(a.w);
        f[4] = __uint_as_float(b.x); f[5] = __uint_as_float(b.y); f[6] = __uint_as_float(b.z); f[7] = __uint_as_float(b.w);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = e0 + j < H ? to_float<T>(p[j]) : 0.f;
    }
  } else {
    const uint8_t* p = static_cast<const uint8_t*>(row) + e0;
    uint32_t w[2] = {0u, 0u};
    if (vec) {
      const uint2 r = *reinterpret_cast<const uint2*>(p);
      w[0] = r.x;
      w[1] = r.y;
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (e0 + j < H) w[j / 4] |= static_cast<uint32_t>(p[j]) << (8 * (j % 4));
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v = rnd<T>(__fmul_rn(s_in, decode8<IN>(w[j / 4] >> (8 * (j % 4)))));
      f[j] = e0 + j < H ? v : 0.f;
    }
  }
}

// gamma / beta chunk, or the identity value when the tensor is absent
template <typename T>
__device__ __forceinline__ void load_param(const T* __restrict__ p, int e0, int H, bool vec, float none, float (&f)[8]) {
  if (p == nullptr) {
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = none;
    return;
  }
  load_chunk<T, kFloatIO>(p, e0, H, vec, 0.f, f);
}

template <typename T, int OUT>
__device__ __forceinline__ void store_chunk(void* __restrict__ row, int e0, int H, bool vec, const float (&y)[8],
                                            float os, float r, bool use_rcp) {
  if constexpr (OUT == kFloatIO) {
    T* p = static_cast<T*>(row) + e0;
    if (vec) {
      if constexpr (sizeof(T) == 2) {
        uint4 o;
        T* e = reinterpret_cast<T*>(&o);
#pragma unroll
        for (int j = 0; j < 8; ++j) e[j] = from_float<T>(y[j]);
        *reinterpret_cast<uint4*>(p) = o;
      } else {
        reinterpret_cast<uint4*>(p)[0] = make_uint4(__float_as_uint(y[0]), __float_as_uint(y[1]), __float_as_uint(y[2]),
                                                    __float_as_uint(y[3]));
        reinterpret_cast<uint4*>(p)[1] = make_uint4(__float_as_uint(y[4]), __float_as_uint(y[5]), __float_as_uint(y[6]),
                                                    __float_as_uint(y[7]));
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (e0 + j < H) p[j] = from_float<T>(y[j]);
    }
  } else {
    uint32_t w[2] = {0u, 0u};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float t = rnd<T>(use_rcp ? __fmul_rn(y[j], r) : __fdiv_rn(y[j], os));
      w[j / 4] |= static_cast<uint32_t>(quantize_one<OUT>(t)) << (8 * (j % 4));
    }
    uint8_t* p = static_cast<uint8_t*>(row) + e0;
    if (vec) {
      *reinterpret_cast<uint2*>(p) = make_uint2(w[0], w[1]);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j)
        if (e0 + j < H) p[j] = static_cast<uint8_t>(w[j / 4] >> (8 * (j % 4)));
    }
  }
}

// sum of v over the row's threads, the same value in every one of them (a fixed order: deterministic)
template <bool WARP>
__device__ __forceinline__ float row_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
  if constexpr (WARP) {
    return v;
  } else {
    const int nw = blockDim.x >> 5;
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float s = red[0];
    for (int w = 1; w < nw; ++w) s = __fadd_rn(s, red[w]);
    return s;
  }
}

template <typename T, int IN, int OUT, bool WARP>
__global__ void __launch_bounds__(WARP ? kWarpThreads : kMaxThreads)
    layernorm_kernel(const void* __restrict__ x, const T* __restrict__ in_scale, const T* __restrict__ gamma,
                     const T* __restrict__ beta, const void* __restrict__ out_scale, bool out_scale_f32,
                     void* __restrict__ out, int64_t rows, int H, float eps, bool vec) {
  __shared__ float red[2][kMaxThreads / 32];
  constexpr int in_bytes = IN == kFloatIO ? static_cast<int>(sizeof(T)) : 1;
  constexpr int out_bytes = OUT == kFloatIO ? static_cast<int>(sizeof(T)) : 1;
  const int G = WARP ? 32 : static_cast<int>(blockDim.x);
  const int gt = WARP ? static_cast<int>(threadIdx.x & 31) : static_cast<int>(threadIdx.x);
  const int64_t per_cta = WARP ? blockDim.x / 32 : 1;
  const int64_t first = WARP ? blockIdx.x * per_cta + threadIdx.x / 32 : blockIdx.x;
  const int nvec = (H + 7) / 8;
  const float s_in = IN == kFloatIO ? 0.f : to_float<T>(*in_scale);
  float os = 1.f, r = 0.f;
  bool use_rcp = false;
  if constexpr (OUT != kFloatIO) {
    os = out_scale_f32 ? *static_cast<const float*>(out_scale) : to_float<T>(*static_cast<const T*>(out_scale));
    use_rcp = !out_scale_f32 && rcp_is_safe<T>(os);  // the bf16-quotient argument needs a bf16 scale
    r = use_rcp ? __frcp_rn(os) : 0.f;
  }
  for (int64_t row = first; row < rows; row += WARP ? gridDim.x * per_cta : gridDim.x) {
    const char* src = static_cast<const char*>(x) + row * H * in_bytes;
    char* dst = static_cast<char*>(out) + row * H * out_bytes;
    float c[kCacheVecs][8];
    float f[8];
    // pass 1: the mean
    float acc = 0.f;
#pragma unroll
    for (int i = 0; i < kCacheVecs; ++i) {
      const int v = gt + i * G;
      if (v < nvec) {
        load_chunk<T, IN>(src, 8 * v, H, vec, s_in, c[i]);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc = __fadd_rn(acc, c[i][j]);
      }
    }
    for (int v = gt + kCacheVecs * G; v < nvec; v += G) {
      load_chunk<T, IN>(src, 8 * v, H, vec, s_in, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc = __fadd_rn(acc, f[j]);
    }
    const float mean = __fdiv_rn(row_sum<WARP>(acc, red[0]), static_cast<float>(H));
    // pass 2: the biased variance about the mean
    acc = 0.f;
#pragma unroll
    for (int i = 0; i < kCacheVecs; ++i) {
      const int v = gt + i * G;
      if (v < nvec) {
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = 8 * v + j < H ? __fsub_rn(c[i][j], mean) : 0.f;
          acc = __fmaf_rn(d, d, acc);
        }
      }
    }
    for (int v = gt + kCacheVecs * G; v < nvec; v += G) {
      load_chunk<T, IN>(src, 8 * v, H, vec, s_in, f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = 8 * v + j < H ? __fsub_rn(f[j], mean) : 0.f;
        acc = __fmaf_rn(d, d, acc);
      }
    }
    const float var = __fdiv_rn(row_sum<WARP>(acc, red[1]), static_cast<float>(H));
    const float rstd = __frsqrt_rn(__fadd_rn(var, eps));
    // pass 3: normalize, scale, shift, round to T, quantize
    auto emit = [&](int v, const float (&xv)[8]) {
      float g[8], b[8], y[8];
      load_param<T>(gamma, 8 * v, H, vec, 1.f, g);
      load_param<T>(beta, 8 * v, H, vec, 0.f, b);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float n = __fmul_rn(__fsub_rn(xv[j], mean), rstd);
        y[j] = rnd<T>(__fmaf_rn(n, g[j], b[j]));
      }
      store_chunk<T, OUT>(dst, 8 * v, H, vec, y, os, r, use_rcp);
    };
#pragma unroll
    for (int i = 0; i < kCacheVecs; ++i) {
      const int v = gt + i * G;
      if (v < nvec) emit(v, c[i]);
    }
    for (int v = gt + kCacheVecs * G; v < nvec; v += G) {
      load_chunk<T, IN>(src, 8 * v, H, vec, s_in, f);
      emit(v, f);
    }
    if constexpr (!WARP) __syncthreads();  // red is rewritten by the next row
  }
}

// the input or output dtype `io`: kFloatIO when it is the float dtype itself, else an 8-bit code dtype ->
// std::integral_constant
template <class F>
int dispatch_ln_io(int io, int dtype, F&& f) {
  if (io == dtype) return f(std::integral_constant<int, kFloatIO>{});
  return dispatch_code8(io, f);
}

// threads of the CTA that owns a row of nvec 8-element chunks: enough to keep the row in registers, at most kMaxThreads
inline int ln_cta_threads(int64_t nvec) {
  const int64_t per = (nvec + kCacheVecs - 1) / kCacheVecs;
  const int64_t t = (per + 31) / 32 * 32;
  return static_cast<int>(t < 64 ? 64 : (t > kMaxThreads ? kMaxThreads : t));
}

}  // namespace qb

using namespace qb;

extern "C" {

int qb200_layer_norm(const void* x, const void* in_scale, const void* weight, const void* bias, const void* out_scale,
                     void* out, int64_t rows, int64_t h, double eps, int in_dtype, int dtype, int out_dtype,
                     int out_scale_dtype, void* stream) {
  set_kernel_family(0);
  if (rows < 0 || h <= 0 || h > INT32_MAX) return fail(ERR_ARG, "layer_norm: bad shape (rows %lld, H %lld)",
                                                       static_cast<long long>(rows), static_cast<long long>(h));
  if (!is_float_dtype(dtype)) return fail(ERR_ARG, "layer_norm: dtype must be F32, F16 or BF16 (got %d)", dtype);
  if (in_dtype != dtype && !is_code_dtype(in_dtype))
    return fail(ERR_ARG, "layer_norm: input dtype %d is neither the float dtype nor an 8-bit code dtype", in_dtype);
  if (out_dtype != dtype && !is_code_dtype(out_dtype))
    return fail(ERR_ARG, "layer_norm: output dtype %d is neither the float dtype nor an 8-bit code dtype", out_dtype);
  if (in_dtype != dtype && in_scale == nullptr) return fail(ERR_ARG, "layer_norm: codes in need their scale");
  if (out_dtype != dtype) {
    if (out_scale == nullptr) return fail(ERR_ARG, "layer_norm: codes out need the output scale");
    if (out_scale_dtype != DT_F32 && out_scale_dtype != dtype)
      return fail(ERR_ARG, "layer_norm: the output scale must be F32 or the float dtype (got %d)", out_scale_dtype);
  }
  if (!(eps >= 0.0)) return fail(ERR_ARG, "layer_norm: eps must be >= 0");
  if (rows == 0) return OK;
  int rc = check_arch("layer_norm");
  if (rc != OK) return rc;
  set_kernel_family(6);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool out_scale_f32 = out_scale_dtype == DT_F32;
  const float e = static_cast<float>(eps);
  const int64_t nvec = (h + 7) / 8;
  const bool vec = h % 8 == 0 && aligned16(x) && aligned16(out) && (weight == nullptr || aligned16(weight)) &&
                   (bias == nullptr || aligned16(bias));
  const bool warp = nvec <= 32 * kCacheVecs;
  const int threads = warp ? kWarpThreads : ln_cta_threads(nvec);
  const int64_t ctas = warp ? (rows + kWarpThreads / 32 - 1) / (kWarpThreads / 32) : rows;
  const unsigned grid = static_cast<unsigned>(ctas < (1 << 20) ? ctas : (1 << 20));
  return dispatch_float(dtype, [&](auto dt) {
    return dispatch_ln_io(in_dtype, dtype, [&](auto IN) {
      return dispatch_ln_io(out_dtype, dtype, [&](auto OUT) {
        using T = typename decltype(dt)::T;
        const auto* sp = static_cast<const T*>(in_scale);
        const auto* gp = static_cast<const T*>(weight);
        const auto* bp = static_cast<const T*>(bias);
        if (warp)
          layernorm_kernel<T, IN.value, OUT.value, true><<<grid, threads, 0, st>>>(
              x, sp, gp, bp, out_scale, out_scale_f32, out, rows, static_cast<int>(h), e, vec);
        else
          layernorm_kernel<T, IN.value, OUT.value, false><<<grid, threads, 0, st>>>(
              x, sp, gp, bp, out_scale, out_scale_f32, out, rows, static_cast<int>(h), e, vec);
        return check_cuda(cudaGetLastError(), "layer_norm launch");
      });
    });
  });
}

}  // extern "C"
