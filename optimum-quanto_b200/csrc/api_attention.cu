// The two kernels that keep per-tensor quantized activations quantized through attention (the reference's
// ActivationQBytesTensor table, optimum/quanto/tensor/activations/qbytes_ops.py):
//
//   qb200_qbytes_bmm      int8 x int8 batched matmul, out[b] = rnd_dt(f32(A[b] @ B[b]) * f32(rnd_dt(sA * sB)))  (:175-186)
//                         on the batched configuration of the wgmma GEMM (gemm_tc.cuh, GemmCfg::BATCH).  wgmma takes
//                         s8 operands K-major only, so a B that arrives N-contiguous (v, or k^T after matmul's reshape)
//                         is first copied K-major by one byte-transpose pass into a caller-provided workspace.  Shapes the
//                         tensor cores do not take run on a batched CUDA-core kernel with the same exact integer sum.
//   qb200_qbytes_softmax  softmax over the last dim of a quantized tensor, re-quantized with the scale 1 / qmax
//                         (:208-215) in one launch: 8-bit codes in, 8-bit codes out.
#include "../../include/quanto_b200.h"

#include "gemm_tc.cuh"
#include "host_common.cuh"

namespace qb {

// ------------------------------------------------------------------------------------------------
// B -> K-major copy: dst[b][n][k] = B[b](k, n), element (k, n) of batch b at src[b * bs + k * sk + n * sn].
// 64 x 64 byte tiles through shared memory; 4-byte loads along n when B is N-contiguous and aligned, 4-byte stores
// along k (K % 16 == 0 on this path).
// ------------------------------------------------------------------------------------------------
constexpr int kTT = 64;

__global__ void __launch_bounds__(256)
    kmajor_copy_kernel(const uint8_t* __restrict__ src, uint8_t* __restrict__ dst, int K, int N, int64_t bs, int64_t sk,
                       int64_t sn, int batches, bool vec) {
  __shared__ __align__(16) uint8_t tile[kTT][kTT + 4];  // [k][n]
  const int n0 = blockIdx.x * kTT, k0 = blockIdx.y * kTT;
  const int t = threadIdx.x;
  for (int b = blockIdx.z; b < batches; b += gridDim.z) {
    const uint8_t* s = src + static_cast<int64_t>(b) * bs;
    if (vec) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int kk = t / 16 + 16 * i, nn = (t % 16) * 4;
        uint32_t w = 0;
        if (k0 + kk < K && n0 + nn < N) w = __ldg(reinterpret_cast<const uint32_t*>(s + (k0 + kk) * sk + n0 + nn));
        *reinterpret_cast<uint32_t*>(&tile[kk][nn]) = w;
      }
    } else {
      for (int i = t; i < kTT * kTT; i += 256) {
        const int kk = i / kTT, nn = i % kTT;
        tile[kk][nn] = (k0 + kk < K && n0 + nn < N) ? s[(k0 + kk) * sk + (n0 + nn) * sn] : 0;
      }
    }
    __syncthreads();
    uint8_t* d = dst + static_cast<int64_t>(b) * N * K;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int nn = t / 16 + 16 * i, kk = (t % 16) * 4;
      if (n0 + nn < N && k0 + kk < K) {
        const uint32_t w = static_cast<uint32_t>(tile[kk][nn]) | (static_cast<uint32_t>(tile[kk + 1][nn]) << 8) |
                           (static_cast<uint32_t>(tile[kk + 2][nn]) << 16) | (static_cast<uint32_t>(tile[kk + 3][nn]) << 24);
        *reinterpret_cast<uint32_t*>(d + static_cast<int64_t>(n0 + nn) * K + k0 + kk) = w;
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// Batched int8 x int8 on CUDA cores, any K, any layout and alignment: the exact int32 sum, then the reference's one fp32
// multiply by rnd_dt(sA * sB) and one rounding to dt.  A[b] is [M, K] row-major at a + b * a_bs.
// ------------------------------------------------------------------------------------------------
constexpr int kST = 64, kSK = 16;

template <typename T>
__global__ void __launch_bounds__(256)
    qbytes_bmm_simt_kernel(const int8_t* __restrict__ A, const int8_t* __restrict__ B, const void* sa, const void* sb,
                           int dt, T* __restrict__ out, int M, int N, int K, int64_t a_bs, int64_t b_bs, int64_t b_sk,
                           int64_t b_sn) {
  __shared__ int s_a[kSK][kST + 1];
  __shared__ int s_b[kSK][kST + 1];
  const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
  const int m0 = blockIdx.y * kST, n0 = blockIdx.x * kST;
  const float scale = scalar_scale_product(sa, sb, dt);
  const int b = blockIdx.z;  // one batch per CTA column
  const int8_t* a = A + static_cast<int64_t>(b) * a_bs;
  const int8_t* w = B + static_cast<int64_t>(b) * b_bs;
  int acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0;
  for (int k0 = 0; k0 < K; k0 += kSK) {
    for (int e = threadIdx.x; e < kST * kSK; e += 256) {
      const int r = e / kSK, kk = e % kSK, k = k0 + kk;
      s_a[kk][r] = (k < K && m0 + r < M) ? a[static_cast<int64_t>(m0 + r) * K + k] : 0;
      s_b[kk][r] = (k < K && n0 + r < N) ? w[k * b_sk + (n0 + r) * b_sn] : 0;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kSK; ++kk) {
      int x[4], y[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { x[i] = s_a[kk][ty * 4 + i]; y[i] = s_b[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] += x[i] * y[j];
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int m = m0 + ty * 4 + i, n = n0 + tx * 4 + j;
      if (m < M && n < N)
        out[(static_cast<int64_t>(b) * M + m) * N + n] = from_float<T>(__fmul_rn(__int2float_rn(acc[i][j]), scale));
    }
}

// the batched configuration of the int8 x int8 wgmma GEMM (int8 only)
template <int MWG, int BN>
using BmmCfg = GemmCfg<MmaKind::I8, BSrc::TMA, MWG, BN, __nv_bfloat16, false, 0, 0, true>;

static bool bmm_tc_shape_ok(const void* a, int64_t m, int64_t n, int64_t k, int64_t a_bs) {
  return k % 16 == 0 && aligned16(a) && a_bs % 16 == 0 && m <= INT32_MAX &&
         n <= INT32_MAX && k <= INT32_MAX;
}

// B needs the K-major copy: it is N-contiguous (or the test route asks for the copy of any layout)
static bool bmm_needs_copy(int b_layout) {
  return b_layout == 1 || test_override(OVR_BMM_ROUTE) == ROUTE_BMM_TRANSPOSE;
}

static int64_t bmm_copy_bytes(int64_t batch, int64_t n, int64_t k, int64_t b_bs) {
  return (b_bs == 0 ? 1 : batch) * n * k;
}

static int qbytes_bmm_impl(const void* a, const void* b, const void* sa, const void* sb, void* out, void* ws,
                           int64_t ws_bytes, int64_t batch, int64_t m, int64_t n, int64_t k, int64_t a_bs, int64_t b_bs,
                           int b_layout, int dt, cudaStream_t st) {
  set_kernel_family(0);
  if (batch < 0 || m < 0 || n < 0 || k <= 0 || a_bs < 0 || b_bs < 0) return fail(ERR_ARG, "qbytes_bmm: bad shape");
  if (b_layout != 0 && b_layout != 1) return fail(ERR_ARG, "qbytes_bmm: b_layout must be 0 (K-contiguous) or 1 (N-contiguous)");
  if (!is_float_dtype(dt)) return fail(ERR_ARG, "qbytes_bmm: scale dtype must be floating point");
  if (sa == nullptr || sb == nullptr) return fail(ERR_ARG, "qbytes_bmm: scales missing");
  if (m > INT32_MAX || n > INT32_MAX || k > INT32_MAX || batch > INT32_MAX)
    return fail(ERR_UNSUPPORTED, "qbytes_bmm: dimension too large");
  if (batch == 0 || m == 0 || n == 0) return OK;
  int rc = check_arch("qbytes_bmm");
  if (rc != OK) return rc;
  const int route = test_override(OVR_BMM_ROUTE);
  const bool copy = bmm_needs_copy(b_layout);
  const bool b_in_place_ok = aligned16(b) && b_bs % 16 == 0;
  const int tile_m = wgmma_tile_m(m);
  const int64_t mb = (m + tile_m - 1) / tile_m;
  if (route != ROUTE_BMM_SIMT && bmm_tc_shape_ok(a, m, n, k, a_bs) && (copy || b_in_place_ok) &&
      batch * ((n + 127) / 128) * mb <= INT32_MAX) {
    const void* bk = b;
    int64_t bk_bs = b_bs;
    if (copy) {
      if (ws == nullptr || ws_bytes < bmm_copy_bytes(batch, n, k, b_bs) || !aligned16(ws))
        return fail(ERR_ARG, "qbytes_bmm: the K-major copy of B needs qb200_qbytes_bmm_workspace_bytes() bytes of "
                             "16-byte aligned workspace");
      const int copies = b_bs == 0 ? 1 : static_cast<int>(batch);
      const int64_t sk = b_layout == 0 ? 1 : n, sn = b_layout == 0 ? k : 1;
      const bool vec = sn == 1 && n % 4 == 0 && reinterpret_cast<uintptr_t>(b) % 4 == 0 && b_bs % 4 == 0;
      dim3 grid(static_cast<unsigned>((n + kTT - 1) / kTT), static_cast<unsigned>((k + kTT - 1) / kTT),
                static_cast<unsigned>(copies < 65535 ? copies : 65535));
      kmajor_copy_kernel<<<grid, 256, 0, st>>>(static_cast<const uint8_t*>(b), static_cast<uint8_t*>(ws),
                                               static_cast<int>(k), static_cast<int>(n), b_bs, sk, sn, copies, vec);
      rc = check_cuda(cudaGetLastError(), "qbytes_bmm K-major copy launch");
      if (rc != OK) return rc;
      bk = ws;
      bk_bs = b_bs == 0 ? 0 : n * k;
    }
    // tile N 256 (A read half as often) when it costs no more waves than 128, as qbytes_mm chooses
    const int64_t sms = current_sm_count();
    auto waves = [&](int bn) { return ((batch * mb * ((n + bn - 1) / bn) + sms - 1) / sms) * bn; };
    int bn = (tile_m == 128 && waves(256) <= waves(128)) ? 256 : 128;
    const int force_bn = test_override(OVR_QBYTES_TILE_N);
    if (force_bn == 128 || force_bn == 256) bn = force_bn;
    GemmParams p = dense_gemm_params(out, nullptr, dt, m, n, k);
    p.scales = sa;
    p.scale_b = sb;
    p.num_m_blocks = static_cast<int>(mb);
    p.n_blocks_per_batch = static_cast<int>((n + bn - 1) / bn);
    p.num_n_blocks = static_cast<int>(batch) * p.n_blocks_per_batch;
    p.a_batch_mul = a_bs == 0 ? 0 : 1;
    p.b_batch_mul = bk_bs == 0 ? 0 : 1;
    CUtensorMap ta, tb;
    rc = make_tmap_3d_bytes(&ta, a, a_bs == 0 ? 1 : batch, m, k, a_bs == 0 ? m * k : a_bs, tile_m);
    if (rc != OK) return rc;
    rc = make_tmap_3d_bytes(&tb, bk, bk_bs == 0 ? 1 : batch, n, k, bk_bs == 0 ? n * k : bk_bs, bn);
    if (rc != OK) return rc;
    set_kernel_family(copy ? 4 : 1);
    return dispatch_mwg(tile_m, [&](auto MWG) {
      if (bn == 256) return launch_gemm_tc<BmmCfg<MWG, 256>>(&ta, &tb, nullptr, p, st, "qbytes_bmm wgmma launch");
      return launch_gemm_tc<BmmCfg<MWG, 128>>(&ta, &tb, nullptr, p, st, "qbytes_bmm wgmma launch");
    });
  }
  if (batch > 65535 || (m + kST - 1) / kST > 65535)
    return fail(ERR_UNSUPPORTED, "qbytes_bmm: the CUDA-core kernel takes at most 65535 batches of 65535 x 64 rows");
  set_kernel_family(2);
  const int64_t b_sk = b_layout == 0 ? 1 : n, b_sn = b_layout == 0 ? k : 1;
  dim3 grid(static_cast<unsigned>((n + kST - 1) / kST), static_cast<unsigned>((m + kST - 1) / kST),
            static_cast<unsigned>(batch));
  return dispatch_float(dt, [&](auto out_dt) {
    using T = typename decltype(out_dt)::T;
    qbytes_bmm_simt_kernel<T><<<grid, 256, 0, st>>>(static_cast<const int8_t*>(a), static_cast<const int8_t*>(b), sa, sb,
                                                    dt, static_cast<T*>(out), static_cast<int>(m), static_cast<int>(n),
                                                    static_cast<int>(k), a_bs, b_bs, b_sk, b_sn);
    return check_cuda(cudaGetLastError(), "qbytes_bmm CUDA-core launch");
  });
}

// ------------------------------------------------------------------------------------------------
// Quantized softmax over rows of `cols` codes, one CTA per row:
//   x = rnd_dt(s * payload)                       QBytesTensor.dequantize (tensor/qbytes.py:23-31)
//   y = rnd_dt(exp(x - max) / sum exp(x - max))   fp32 max, exp and sum (aten._softmax in dt)
//   q = quantize_symmetric(y, qtype, 1 / qmax)    quantize_math.cuh, the scale rounded to dt by the caller
// Pass 1 keeps a running (max, sum) per thread, rescaling the sum when the max grows; pass 2 writes the codes.  A row
// of up to kSmCache codes is kept in shared memory between the two passes (read from memory once); a longer row is
// read twice.
// ------------------------------------------------------------------------------------------------
constexpr int kSmThreads = 128;
constexpr int kSmCache = 32768;

// (m, s) <- the running (max, sum) of the union of two sets of values
__device__ __forceinline__ void softmax_merge(float& m, float& s, float m2, float s2) {
  if (s2 == 0.f) return;
  if (s == 0.f) {
    m = m2;
    s = s2;
    return;
  }
  const float mn = fmaxf(m, m2);
  s = s * expf(m - mn) + s2 * expf(m2 - mn);
  m = mn;
}

__device__ __forceinline__ uint32_t load_codes4(const uint8_t* row, int64_t e, int64_t cols, bool vec) {
  if (vec) return __ldcs(reinterpret_cast<const unsigned int*>(row + e));
  uint32_t w = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (e + j < cols) w |= static_cast<uint32_t>(row[e + j]) << (8 * j);
  return w;
}

template <typename T, int Q>
__global__ void __launch_bounds__(kSmThreads)
    qbytes_softmax_kernel(const uint8_t* __restrict__ x, const T* __restrict__ scale, const T* __restrict__ out_scale,
                          uint8_t* __restrict__ out, int64_t rows, int64_t cols) {
  __shared__ __align__(16) uint8_t cache[kSmCache];
  __shared__ float red_m[kSmThreads / 32], red_s[kSmThreads / 32];
  const float s = to_float<T>(*scale);
  const float os = to_float<T>(*out_scale);
  const bool use_rcp = rcp_is_safe<T>(os);
  const float r = use_rcp ? __frcp_rn(os) : 0.f;
  const bool cached = cols <= kSmCache;
  const bool vec = cols % 4 == 0 && reinterpret_cast<uintptr_t>(x) % 4 == 0 && reinterpret_cast<uintptr_t>(out) % 4 == 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const uint8_t* src = x + row * cols;
    uint8_t* dst = out + row * cols;
    float m = -INFINITY, sum = 0.f;
    for (int64_t e = 4 * static_cast<int64_t>(threadIdx.x); e < cols; e += 4 * kSmThreads) {
      const uint32_t w = load_codes4(src, e, cols, vec);
      if (cached) *reinterpret_cast<uint32_t*>(cache + e) = w;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (e + j >= cols) break;
        const float v = rnd<T>(__fmul_rn(s, decode8<Q>(w >> (8 * j))));
        if (v == -INFINITY) continue;  // contributes exp(-inf) = 0 (and must not meet a max of -inf)
        if (v > m) {
          sum = sum * expf(m - v) + 1.f;
          m = v;
        } else {
          sum += expf(v - m);
        }
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, sum, o);
      softmax_merge(m, sum, m2, s2);
    }
    if (lane == 0) {
      red_m[warp] = m;
      red_s[warp] = sum;
    }
    __syncthreads();
    m = red_m[0];
    sum = red_s[0];
#pragma unroll
    for (int w = 1; w < kSmThreads / 32; ++w) softmax_merge(m, sum, red_m[w], red_s[w]);
    for (int64_t e = 4 * static_cast<int64_t>(threadIdx.x); e < cols; e += 4 * kSmThreads) {
      const uint32_t w = cached ? *reinterpret_cast<const uint32_t*>(cache + e) : load_codes4(src, e, cols, vec);
      uint32_t q4 = 0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float v = rnd<T>(__fmul_rn(s, decode8<Q>(w >> (8 * j))));
        const float y = rnd<T>(__fdiv_rn(expf(v - m), sum));
        const float t = rnd<T>(use_rcp ? __fmul_rn(y, r) : __fdiv_rn(y, os));
        q4 |= static_cast<uint32_t>(quantize_one<Q>(t)) << (8 * j);
      }
      if (vec) {
        __stcs(reinterpret_cast<unsigned int*>(dst + e), q4);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (e + j < cols) dst[e + j] = static_cast<uint8_t>(q4 >> (8 * j));
      }
    }
    __syncthreads();  // red_m / red_s and the cache are rewritten by the next row
  }
}

}  // namespace qb

using namespace qb;

extern "C" {

int64_t qb200_qbytes_bmm_workspace_bytes(int64_t batch, int64_t n, int64_t k, int64_t b_batch_stride, int b_layout) {
  if (batch <= 0 || n <= 0 || k <= 0 || !bmm_needs_copy(b_layout)) return 0;
  return bmm_copy_bytes(batch, n, k, b_batch_stride);
}

int qb200_qbytes_bmm(const void* a, const void* b, const void* scale_a, const void* scale_b, void* out, void* workspace,
                     int64_t workspace_bytes, int64_t batch, int64_t m, int64_t n, int64_t k, int64_t a_batch_stride,
                     int64_t b_batch_stride, int b_layout, int scale_dtype, void* stream) {
  return qbytes_bmm_impl(a, b, scale_a, scale_b, out, workspace, workspace_bytes, batch, m, n, k, a_batch_stride,
                         b_batch_stride, b_layout, scale_dtype, static_cast<cudaStream_t>(stream));
}

int qb200_qbytes_softmax(const void* x, const void* scale, const void* out_scale, void* out, int64_t rows, int64_t cols,
                         int q_dtype, int scale_dtype, void* stream) {
  if (rows < 0 || cols <= 0) return fail(ERR_ARG, "qbytes_softmax: bad shape");
  if (!is_code_dtype(q_dtype)) return fail(ERR_ARG, "qbytes_softmax: unsupported code dtype %d", q_dtype);
  if (scale == nullptr || out_scale == nullptr) return fail(ERR_ARG, "qbytes_softmax: scales missing");
  if (rows == 0) return OK;
  if (!is_float_dtype(scale_dtype)) return fail(ERR_ARG, "qbytes_softmax: scale dtype must be floating point");
  int rc = check_arch("qbytes_softmax");
  if (rc != OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const unsigned grid = static_cast<unsigned>(rows < (1 << 20) ? rows : (1 << 20));
  return dispatch_float(scale_dtype, [&](auto dt) {
    return dispatch_code8(q_dtype, [&](auto Q) {
      using T = typename decltype(dt)::T;
      qbytes_softmax_kernel<T, Q><<<grid, kSmThreads, 0, st>>>(static_cast<const uint8_t*>(x), static_cast<const T*>(scale),
                                                               static_cast<const T*>(out_scale),
                                                               static_cast<uint8_t*>(out), rows, cols);
      return check_cuda(cudaGetLastError(), "qbytes_softmax launch");
    });
  });
}

}  // extern "C"
