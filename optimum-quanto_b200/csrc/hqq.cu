// HQQ weight optimizer (optimum/quanto/tensor/optimizers/hqq_optimizer.py:28-34 shrink_lp_op, :60-87 optimize) fused
// with quantize_affine + pack_weights for an axis-0 int4 / int2 weight: two launches, no host synchronisation.
//
//   hqq_search_kernel  each grouped row [G] is held in registers by a team of G/8 lanes (freeze.cu's layout) and
//                      runs the ALL-ACCEPTED trajectory for `iters` steps.  beta only changes on acceptance and the loop
//                      stops at the first rejection, so every row's candidate shifts are fixed in advance; the only
//                      global quantity is the stop index.  Each step's candidate shift is stored per row, each step's
//                      |base - dequant| sum goes to a per-CTA fp64 partial, and the last CTA to finish (ticket, as in
//                      absmax) sums the partials in CTA order, rounds each mean to the weight dtype and applies the stop
//                      rule.  Deterministic: fixed grid, fixed row-to-CTA assignment, fixed reduction orders.
//   hqq_pack_kernel    one team per packed row: reads the accepted shift, writes the shift (or uint8 zero-point) and
//                      the canonical packed codes of every bit plane.
//
// Every step follows the rounding order of the reference on CPU tensors (DESIGN.md §4):
//   dequant  : rnd(rnd(q * s) - z)                                              (QBitsDequantizer, two roundings)
//   shrink   : rnd(|x| - rnd(fp32(1/beta) * rnd(pow(|x|, e_dt))))  or  rnd(|x| - rnd(fp32(1/beta))) for lp == 1;
//              relu keeps NaN, sign(NaN) = sign(0) = 0
//   candidate: rnd_dt(sum_fp64(rnd(rnd(q * s) - rnd(b - e))) / G)               (torch.mean rounds once)
//   requant  : quantize_affine's float-shift path (quantize_math.cuh)
//   error    : rnd_dt(sum_fp64 |rnd(b - dequant)| / (N*K)), compared after rounding (ties stop the loop)
// pow(|x|, e_dt) comes from a 32768-entry table of the dtype's magnitudes, built per CTA in shared memory as
// rnd_dt(rnd_f32(pow_f64)): the float32 power rounded to the dtype, which is what torch's CPU pow returns.
#include <type_traits>

#include "../../include/quanto_b200.h"

#include "host_common.cuh"
#include "quantize_math.cuh"

namespace qb {

constexpr int kHqqThreads = 256;
constexpr int kHqqWarps = kHqqThreads / 32;
constexpr int kHqqMaxIters = 64;
constexpr int kHqqTable = 32768;      // one entry per non-negative 16-bit pattern
constexpr int kHqqCtasPerSm = 2;

struct HqqParams {
  float inv_beta[kHqqMaxIters];  // fp32(1.0 / beta_i), beta_i = beta * kappa^i by repeated double multiplication
};

struct HqqHeader {  // start of the workspace
  unsigned int ticket;  // CTAs of the search launch that have published their partials (zeroed before it)
  int accepted;         // the number of accepted iterations, written by the last CTA
};

template <typename T>
__device__ __forceinline__ unsigned magnitude_bits(float a) {  // a >= 0, exactly representable in T
  const T h = from_float<T>(a);
  return static_cast<unsigned>(*reinterpret_cast<const unsigned short*>(&h)) & 0x7FFFu;
}

template <typename T>
__device__ __forceinline__ float rnd64(double v) {  // one rounding from fp64 to T
  if constexpr (std::is_same<T, __nv_bfloat16>::value) return __bfloat162float(__double2bfloat16(v));
  else return __half2float(__double2half(v));
}

template <typename T>
__device__ void build_pow_table(T* table, double e) {
  for (int i = threadIdx.x; i < kHqqTable; i += blockDim.x) {
    unsigned short u = static_cast<unsigned short>(i);
    const float a = to_float<T>(*reinterpret_cast<const T*>(&u));
    table[i] = from_float<T>(static_cast<float>(pow(static_cast<double>(a), e)));
  }
}

// shrink_lp_op of one value of T; `inv` = fp32(1/beta) (LP1: already rounded to T)
template <typename T, bool LP1>
__device__ __forceinline__ float shrink_one(float x, float inv, const T* table) {
  const float a = fabsf(x);
  float d;
  if constexpr (LP1) {
    d = rnd<T>(__fsub_rn(a, inv));
  } else {
    const float p = to_float<T>(table[magnitude_bits<T>(a)]);
    d = rnd<T>(__fsub_rn(a, rnd<T>(__fmul_rn(inv, p))));
  }
  const float r = d > 0.f ? d : (d != d ? d : 0.f);
  const float sgn = x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f);
  return __fmul_rn(sgn, r);
}

template <typename T, int BITS>
__device__ __forceinline__ void quantize_row8(const float (&b)[8], float s, float r, bool fast, float z, float (&q)[8]) {
  uint32_t codes[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
  if (fast) affine_quantize8<T, false, true>(b, s, r, z, (1 << BITS) - 1, 0, codes);
  else affine_quantize8<T, false, false>(b, s, 0.f, z, (1 << BITS) - 1, 0, codes);
#pragma unroll
  for (int j = 0; j < 8; ++j) q[j] = static_cast<float>(codes[j]);
}

// sum over the lane's 8 values of |rnd(b - rnd(rnd(q * s) - z))|
template <typename T>
__device__ __forceinline__ double abs_error8(const float (&b)[8], const float (&q)[8], float s, float z) {
  double acc = 0.0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float dq = rnd<T>(__fsub_rn(rnd<T>(__fmul_rn(q[j], s)), z));
    acc += static_cast<double>(fabsf(rnd<T>(__fsub_rn(b[j], dq))));
  }
  return acc;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

template <typename T, int BITS, int TL, bool LP1>
__global__ void __launch_bounds__(kHqqThreads)
    hqq_search_kernel(const T* __restrict__ base, T* __restrict__ scale_out, T* __restrict__ cands,
                      double* __restrict__ partials, HqqHeader* __restrict__ header, float* __restrict__ errors,
                      int64_t rows, int group, int iters, double pow_exp, double numel, const HqqParams P) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* table = reinterpret_cast<T*>(smem_raw);
  __shared__ double werr[kHqqWarps][kHqqMaxIters + 1];
  __shared__ float means[kHqqMaxIters + 1];
  __shared__ bool is_last;
  constexpr float QMAX = static_cast<float>((1 << BITS) - 1);
  constexpr int TEAMS_PER_WARP = 32 / TL;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int col0 = (lane % TL) * 8;
  const bool lane_active = col0 < group;
  const bool leader = (lane % TL) == 0;

  if constexpr (!LP1) build_pow_table<T>(table, pow_exp);
  for (int i = threadIdx.x; i < kHqqWarps * (kHqqMaxIters + 1); i += blockDim.x) (&werr[0][0])[i] = 0.0;
  __syncthreads();

  const int64_t warp_global = static_cast<int64_t>(blockIdx.x) * kHqqWarps + warp;
  const int64_t step = static_cast<int64_t>(gridDim.x) * kHqqWarps * TEAMS_PER_WARP;
  for (int64_t r0 = warp_global * TEAMS_PER_WARP; r0 < rows; r0 += step) {  // bound uniform per warp
    const int64_t row = r0 + lane / TL;
    const bool valid = row < rows && lane_active;
    float b[8];
    if (valid) load8_stream<T>(base + row * group + col0, b);
    else
#pragma unroll
      for (int j = 0; j < 8; ++j) b[j] = 0.f;
    // MaxOptimizer: scale = rnd(rnd(hi - lo) / (2^bits - 1)), shift = -lo
    float lo = __int_as_float(0x7f800000), hi = __int_as_float(0xff800000);
    if (valid) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        lo = fminf(lo, b[j]);
        hi = fmaxf(hi, b[j]);
      }
    }
#pragma unroll
    for (int off = TL / 2; off > 0; off >>= 1) {
      lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, off));
      hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, off));
    }
    const float s = rnd<T>(__fdiv_rn(rnd<T>(__fsub_rn(hi, lo)), QMAX));
    const bool fast = rcp_is_safe<T>(s);
    const float rs = fast ? __frcp_rn(s) : 0.f;
    float z = -lo;
    if (row < rows && leader) {
      scale_out[row] = from_float<T>(s);
      cands[row] = from_float<T>(z);
    }
    float q[8];
    quantize_row8<T, BITS>(b, s, rs, fast, z, q);
    double e = warp_sum(valid ? abs_error8<T>(b, q, s, z) : 0.0);
    if (lane == 0) werr[warp][0] += e;
    for (int it = 0; it < iters; ++it) {
      float inv = P.inv_beta[it];
      if constexpr (LP1) inv = rnd<T>(inv);
      double acc = 0.0;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float a = rnd<T>(__fmul_rn(q[j], s));
        const float x = rnd<T>(__fsub_rn(b[j], rnd<T>(__fsub_rn(a, z))));
        const float sh = shrink_one<T, LP1>(x, inv, table);
        acc += static_cast<double>(rnd<T>(__fsub_rn(a, rnd<T>(__fsub_rn(b[j], sh)))));
      }
      if (!valid) acc = 0.0;
#pragma unroll
      for (int off = TL / 2; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
      z = rnd64<T>(acc / static_cast<double>(group));
      if (row < rows && leader) cands[static_cast<int64_t>(it + 1) * rows + row] = from_float<T>(z);
      quantize_row8<T, BITS>(b, s, rs, fast, z, q);
      e = warp_sum(valid ? abs_error8<T>(b, q, s, z) : 0.0);
      if (lane == 0) werr[warp][it + 1] += e;
    }
  }
  __syncthreads();
  if (threadIdx.x <= iters) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < kHqqWarps; ++w) t += werr[w][threadIdx.x];
    partials[static_cast<int64_t>(blockIdx.x) * (iters + 1) + threadIdx.x] = t;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(&header->ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (threadIdx.x <= iters) {
    double t = 0.0;
    for (unsigned c = 0; c < gridDim.x; ++c) t += __ldcg(partials + static_cast<int64_t>(c) * (iters + 1) + threadIdx.x);
    means[threadIdx.x] = rnd64<T>(t / numel);
    errors[threadIdx.x] = means[threadIdx.x];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // the reference's stop rule on the dt-rounded means: accept while strictly below the best so far
    int accepted = 0;
    float best = means[0];
    while (accepted < iters && means[accepted + 1] < best) best = means[++accepted];
    errors[iters + 1] = static_cast<float>(accepted);
    header->accepted = accepted;
  }
}

template <typename T, int BITS, bool ZP, int TL>
__global__ void __launch_bounds__(kHqqThreads)
    hqq_pack_kernel(const T* __restrict__ base, uint8_t* __restrict__ packed, const T* __restrict__ scale,
                    void* __restrict__ shift, const T* __restrict__ cands, const HqqHeader* __restrict__ header,
                    int64_t rows, int64_t packed_rows, int group) {
  constexpr int PLANES = 8 / BITS;
  constexpr int QMAX = (1 << BITS) - 1;
  constexpr int TEAMS_PER_WARP = 32 / TL;
  const int lane = threadIdx.x & 31;
  const int col0 = (lane % TL) * 8;
  const bool lane_active = col0 < group;
  const T* accepted_shift = cands + static_cast<int64_t>(__ldcg(&header->accepted)) * rows;
  const int64_t warp_global = static_cast<int64_t>(blockIdx.x) * kHqqWarps + (threadIdx.x >> 5);
  const int64_t step = static_cast<int64_t>(gridDim.x) * kHqqWarps * TEAMS_PER_WARP;
  for (int64_t pr = warp_global * TEAMS_PER_WARP + lane / TL; pr < packed_rows; pr += step) {
    uint32_t bytes[8] = {0u, 0u, 0u, 0u, 0u, 0u, 0u, 0u};
#pragma unroll
    for (int p = 0; p < PLANES; ++p) {
      const int64_t row = pr + static_cast<int64_t>(p) * packed_rows;
      if (row >= rows) continue;
      const float s = to_float<T>(scale[row]);
      float z = to_float<T>(accepted_shift[row]);
      const bool fast = rcp_is_safe<T>(s);
      const float r = fast ? __frcp_rn(s) : 0.f;
      if constexpr (ZP) {  // AffineOptimizer: clamp(round(shift / scale), 0, 2^bits - 1) as uint8; NaN -> 0
        const float zq = fast ? rnd<T>(__fmul_rn(z, r)) : rnd<T>(__fdiv_rn(z, s));
        z = fminf(fmaxf(rintf(zq), 0.f), static_cast<float>(QMAX));
      }
      if (lane_active) {
        float f[8];
        load8_stream<T>(base + row * group + col0, f);
        if (fast) affine_quantize8<T, ZP, true>(f, s, r, z, QMAX, BITS * p, bytes);
        else affine_quantize8<T, ZP, false>(f, s, 0.f, z, QMAX, BITS * p, bytes);
      }
      if ((lane % TL) == 0) {
        if constexpr (ZP) static_cast<uint8_t*>(shift)[row] = static_cast<uint8_t>(z);
        else static_cast<T*>(shift)[row] = from_float<T>(z);
      }
    }
    if (lane_active) {
      uint2 o;
      o.x = bytes[0] | (bytes[1] << 8) | (bytes[2] << 16) | (bytes[3] << 24);
      o.y = bytes[4] | (bytes[5] << 8) | (bytes[6] << 16) | (bytes[7] << 24);
      __stcs(reinterpret_cast<uint2*>(packed + pr * group + col0), o);
    }
  }
}

template <typename T, bool LP1>
__global__ void __launch_bounds__(kHqqThreads)
    hqq_shrink_kernel(const T* __restrict__ x, T* __restrict__ out, int64_t numel, float inv, double pow_exp) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* table = reinterpret_cast<T*>(smem_raw);
  if constexpr (!LP1) {
    build_pow_table<T>(table, pow_exp);
    __syncthreads();
  } else {
    inv = rnd<T>(inv);
  }
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < numel; i += stride)
    out[i] = from_float<T>(shrink_one<T, LP1>(to_float<T>(x[i]), inv, table));
}

// ----------------------------------------------------------------------------------------------------- host side
static int hqq_search_grid(int64_t rows, int group) {
  return capped_grid(rows, kHqqThreads / team_lanes(group), kHqqCtasPerSm);
}

static size_t align256(size_t b) { return (b + 255) & ~static_cast<size_t>(255); }

struct HqqLayout {
  size_t partials, cands, total;
};

static HqqLayout hqq_layout(int64_t rows, int group, int iters, int elem_bytes) {
  HqqLayout l;
  l.partials = 256;
  l.cands = l.partials + align256(sizeof(double) * hqq_search_grid(rows, group) * static_cast<size_t>(iters + 1));
  l.total = l.cands + align256(static_cast<size_t>(elem_bytes) * rows * static_cast<size_t>(iters + 1));
  return l;
}

// dynamic shared memory of the pow table: none for lp_norm == 1 (LP1), which needs no power
template <typename T, bool LP1>
static int table_smem() {
  return LP1 ? 0 : kHqqTable * static_cast<int>(sizeof(T));
}

// opts `kern` into `smem` bytes of dynamic shared memory when it uses any
template <class Kernel>
static int opt_into_table(Kernel kern, int smem, const char* what) {
  if (smem == 0) return OK;
  return check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem), what);
}

// the pow exponent torch uses: python's lp_norm - 1 converted to the tensor dtype (through float, as c10 does)
template <typename T>
static double hqq_pow_exponent(double lp_norm) {
  return static_cast<double>(static_cast<float>(T(static_cast<float>(lp_norm - 1.0))));
}

// ERR_UNSUPPORTED (the caller composes ATen ops) for what the kernel does not reproduce bit for bit
static int hqq_check_config(const char* what, int dtype, double lp_norm) {
  if (dtype == DT_F32)
    return fail(ERR_UNSUPPORTED, "%s: float32 weights (the reference's float32 pow is not correctly rounded)", what);
  if (dtype != DT_F16 && dtype != DT_BF16) return fail(ERR_ARG, "%s: dtype %d not floating point", what, dtype);
  if (!(lp_norm > 0.0)) return fail(ERR_UNSUPPORTED, "%s: lp_norm must be > 0, got %g", what, lp_norm);
  const double e = dtype == DT_BF16 ? hqq_pow_exponent<__nv_bfloat16>(lp_norm) : hqq_pow_exponent<__half>(lp_norm);
  if (e == 3.0)  // torch computes x * x * x there, which is not the rounded power
    return fail(ERR_UNSUPPORTED, "%s: lp_norm %g (torch.pow special-cases the cube)", what, lp_norm);
  return OK;
}

}  // namespace qb

using namespace qb;

extern "C" {

int64_t qb200_quantize_qbits_hqq_workspace_bytes(int64_t n, int64_t k, int group, int iters) {
  if (n <= 0 || k <= 0 || group <= 0 || k % group != 0 || iters < 0 || iters > kHqqMaxIters) return 0;
  return static_cast<int64_t>(hqq_layout(n * k / group, group, iters, 2).total);
}

int qb200_quantize_qbits_hqq(const void* base, uint8_t* packed, void* scale, void* shift, float* errors,
                             void* workspace, int64_t n, int64_t k, int group, int bits, int dtype, int zeropoint,
                             double lp_norm, double beta, double kappa, int iters, void* stream) {
  const char* what = "quantize_qbits_hqq";
  if (bits != 2 && bits != 4) return fail(ERR_ARG, "%s: bits must be 2 or 4, got %d", what, bits);
  if (n <= 0 || k <= 0 || group <= 0) return fail(ERR_ARG, "%s: bad shape", what);
  if (k % group != 0) return fail(ERR_ARG, "%s: group %d does not divide K=%lld", what, group, (long long)k);
  if (iters < 0) return fail(ERR_ARG, "%s: iters must be >= 0, got %d", what, iters);
  int rc = hqq_check_config(what, dtype, lp_norm);
  if (rc != OK) return rc;
  if (group % 8 != 0 || group > 256)
    return fail(ERR_UNSUPPORTED, "%s: group %d (needs a multiple of 8, <= 256)", what, group);
  if (iters > kHqqMaxIters) return fail(ERR_UNSUPPORTED, "%s: iters %d > %d", what, iters, kHqqMaxIters);
  if (!base || !packed || !scale || !shift || !errors || !workspace) return fail(ERR_ARG, "%s: null buffer", what);
  if (reinterpret_cast<uintptr_t>(base) % 16 != 0 || reinterpret_cast<uintptr_t>(packed) % 8 != 0 ||
      reinterpret_cast<uintptr_t>(workspace) % 256 != 0)
    return fail(ERR_UNSUPPORTED, "%s: base must be 16-byte, packed 8-byte and workspace 256-byte aligned", what);
  const int64_t rows = n * k / group;
  const int64_t packed_rows = (rows + (8 / bits) - 1) / (8 / bits);
  const HqqLayout L = hqq_layout(rows, group, iters, 2);
  char* ws = static_cast<char*>(workspace);
  HqqHeader* header = reinterpret_cast<HqqHeader*>(ws);
  double* partials = reinterpret_cast<double*>(ws + L.partials);
  HqqParams P;
  double b = beta;
  for (int i = 0; i < kHqqMaxIters; ++i) {
    P.inv_beta[i] = static_cast<float>(1.0 / b);
    b *= kappa;
  }
  const double numel = static_cast<double>(n) * static_cast<double>(k);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  rc = check_cuda(cudaMemsetAsync(workspace, 0, sizeof(HqqHeader), st), "quantize_qbits_hqq: workspace memset");
  if (rc != OK) return rc;
  return dispatch_act16(dtype, [&](auto act) {
    return dispatch_bits(bits, [&](auto BITS) {
      return dispatch_team_lanes(group, [&](auto TL) {
        using T = typename decltype(act)::WT;
        T* cands = reinterpret_cast<T*>(ws + L.cands);
        auto search = [&](auto LP1) {
          auto kern = hqq_search_kernel<T, BITS, TL, LP1>;
          const int smem = table_smem<T, LP1>();
          const int set = opt_into_table(kern, smem, "quantize_qbits_hqq: cudaFuncSetAttribute");
          if (set != OK) return set;
          kern<<<hqq_search_grid(rows, group), kHqqThreads, smem, st>>>(
              static_cast<const T*>(base), static_cast<T*>(scale), cands, partials, header, errors, rows, group, iters,
              hqq_pow_exponent<T>(lp_norm), numel, P);
          return check_cuda(cudaGetLastError(), "quantize_qbits_hqq search launch");
        };
        const int searched = lp_norm == 1.0 ? search(std::true_type{}) : search(std::false_type{});
        if (searched != OK) return searched;
        return dispatch_zp(zeropoint, [&](auto ZP) {
          hqq_pack_kernel<T, BITS, ZP, TL><<<capped_grid(packed_rows, kHqqThreads / TL, 8), kHqqThreads, 0, st>>>(
              static_cast<const T*>(base), packed, static_cast<const T*>(scale), shift, cands, header, rows,
              packed_rows, group);
          return check_cuda(cudaGetLastError(), "quantize_qbits_hqq pack launch");
        });
      });
    });
  });
}

int qb200_hqq_shrink(const void* x, void* out, int64_t numel, double beta, double lp_norm, int dtype, void* stream) {
  const char* what = "hqq_shrink";
  if (numel < 0) return fail(ERR_ARG, "%s: negative size", what);
  const int rc = hqq_check_config(what, dtype, lp_norm);
  if (rc != OK) return rc;
  if (numel == 0) return OK;
  if (!x || !out) return fail(ERR_ARG, "%s: null buffer", what);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const float inv = static_cast<float>(1.0 / beta);
  const int grid = capped_grid(numel, kHqqThreads, 2);
  return dispatch_act16(dtype, [&](auto act) {
    using T = typename decltype(act)::WT;
    auto shrink = [&](auto LP1) {
      auto kern = hqq_shrink_kernel<T, LP1>;
      const int smem = table_smem<T, LP1>();
      const int set = opt_into_table(kern, smem, "hqq_shrink: cudaFuncSetAttribute");
      if (set != OK) return set;
      kern<<<grid, kHqqThreads, smem, st>>>(static_cast<const T*>(x), static_cast<T*>(out), numel, inv,
                                           hqq_pow_exponent<T>(lp_norm));
      return check_cuda(cudaGetLastError(), "hqq_shrink launch");
    };
    return lp_norm == 1.0 ? shrink(std::true_type{}) : shrink(std::false_type{});
  });
}

}  // extern "C"
