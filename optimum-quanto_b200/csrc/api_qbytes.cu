// qb200_qbytes_mm / qb200_qbytes_mm_quantized: argument checks, kernel selection and the instantiations of the 8-bit
// paths: int8 x int8 on wgmma with both operands fed by TMA (gemm_tc.cuh), fp8 x fp8 and weight-only fp16 / bf16 x
// int8 / fp8 with the conversion to 16 bits in the staging warps, and the shape-agnostic CUDA-core kernel.
#include "../../include/quanto_b200.h"

#include <cstring>

#include "gemm_tc.cuh"
#include "host_common.cuh"

namespace qb {

int launch_qbytes_mm_simt(const void*, const void*, const void*, const void*, void*, int, int, int, int, int, int,
                          cudaStream_t);

template <class Cfg>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  CUtensorMap tout;
  std::memset(&tout, 0, sizeof(tout));  // the 8-bit epilogues store straight from the accumulators
  return launch_persistent<gemm_tc_kernel<Cfg>, typename Cfg::Pipe>(p.num_m_blocks * p.num_n_blocks, stream,
                                                                    "gemm_tc_kernel launch", ta, tb, tout, p);
}

// Columns of tensor-core work per SM for a tile of BM x bn: waves x bn (wave quantisation included).
static int64_t wave_cost(int64_t m, int64_t n, int bm, int bn) {
  const int64_t tiles = ((m + bm - 1) / bm) * ((n + bn - 1) / bn);
  const int64_t sms = current_sm_count();
  return ((tiles + sms - 1) / sms) * bn;
}

template <int MWG, int BN>
static int launch_int8(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t st) {
  return launch_gemm<GemmCfg<MmaKind::I8, BSrc::TMA, MWG, BN>>(ta, tb, p, st);
}

// fp8 x fp8: both operands converted to bf16 by the staging warps (exact), bf16 MMAs with fp32 accumulation.  Hopper's
// native fp8 MMA accumulates with fewer bits than fp32 and misses the exact-product / fp32-sum contract.
template <int MWG>
static int launch_fp8(int a_dt, int w_dt, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p,
                      cudaStream_t st) {
  constexpr int BN = 128, E4 = 1, E5 = 2;
  using BF = __nv_bfloat16;
  if (a_dt == DT_E4M3 && w_dt == DT_E4M3) return launch_gemm<GemmCfg<MmaKind::BF16, BSrc::F8, MWG, BN, BF, false, E4, E4>>(ta, tb, p, st);
  if (a_dt == DT_E4M3) return launch_gemm<GemmCfg<MmaKind::BF16, BSrc::F8, MWG, BN, BF, false, E5, E4>>(ta, tb, p, st);
  if (w_dt == DT_E4M3) return launch_gemm<GemmCfg<MmaKind::BF16, BSrc::F8, MWG, BN, BF, false, E4, E5>>(ta, tb, p, st);
  return launch_gemm<GemmCfg<MmaKind::BF16, BSrc::F8, MWG, BN, BF, false, E5, E5>>(ta, tb, p, st);
}

// q_dt != 0: the output is quantised in the epilogue (out = [M, N] bytes, q_scale = device pointer to the per-tensor
// output scale in out_dtype); only the int8 x int8 / fp8 x fp8 tensor-core kernels do that.
static int qbytes_mm_impl(const void* a, const void* w, const void* scales, const void* bias, void* out, int64_t m,
                          int64_t n, int64_t k, int a_dtype, int w_dtype, int out_dtype, int q_dt, const void* q_scale,
                          void* stream) {
  set_kernel_family(0);
  if (m < 0 || n <= 0 || k <= 0) return fail(ERR_ARG, "qbytes_mm: bad shape");
  if (out_dtype != DT_F32 && out_dtype != DT_F16 && out_dtype != DT_BF16)
    return fail(ERR_ARG, "qbytes_mm: scales/out dtype must be floating point");
  if (w_dtype != DT_I8 && w_dtype != DT_E4M3 && w_dtype != DT_E5M2 && w_dtype != DT_E4M3FNUZ)
    return fail(ERR_ARG, "qbytes_mm: weights must be int8 or float8");
  if (a_dtype < DT_F32 || a_dtype > DT_E4M3FNUZ || a_dtype == DT_U8) return fail(ERR_ARG, "qbytes_mm: bad activation dtype");
  if (m > INT32_MAX || n > INT32_MAX || k > INT32_MAX) return fail(ERR_UNSUPPORTED, "qbytes_mm: dimension too large");
  if (m == 0) return OK;
  int rc = check_arch();
  if (rc != OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int route = test_override(OVR_QBYTES_ROUTE);

  auto base_params = [&]() {
    GemmParams p{};
    p.bias = bias;
    p.out = out;
    p.g.out_peer[0] = out;
    p.g.n_out = 1;
    p.g.world = 1;
    p.ld = static_cast<int>(n);
    p.col0 = 0;
    p.out_dt = out_dtype;
    p.M = static_cast<int>(m);
    p.N = static_cast<int>(n);
    p.K = static_cast<int>(k);
    return p;
  };
  const int tile_m = wgmma_tile_m(m);

  const bool both_i8 = (a_dtype == DT_I8 && w_dtype == DT_I8);
  const bool both_f8 = ((a_dtype == DT_E4M3 || a_dtype == DT_E5M2) && (w_dtype == DT_E4M3 || w_dtype == DT_E5M2));
  const bool tma_ok = (k % 16 == 0) && (reinterpret_cast<uintptr_t>(a) % 16 == 0) &&
                      (reinterpret_cast<uintptr_t>(w) % 16 == 0) && (reinterpret_cast<uintptr_t>(out) % 16 == 0);
  if ((both_i8 || both_f8) && tma_ok && route != ROUTE_QBYTES_SIMT) {
    GemmParams p = base_params();
    p.scales = scales;
    p.q_dt = q_dt;
    p.q_scale = q_scale;
    // int8: tile N 128 or 256 (the wider tile reads A half as often), picked by wave cost; fp8: 128 (staged operands)
    int bn = 128;
    if (both_i8) {
      bn = (tile_m == 128 && wave_cost(m, n, tile_m, 256) <= wave_cost(m, n, tile_m, 128)) ? 256 : 128;
      const int force_bn = test_override(OVR_QBYTES_TILE_N);
      if (force_bn == 128 || force_bn == 256) bn = force_bn;
    }
    p.num_m_blocks = static_cast<int>((m + tile_m - 1) / tile_m);
    p.num_n_blocks = static_cast<int>((n + bn - 1) / bn);
    CUtensorMap ta, tb;
    std::memset(&ta, 0, sizeof(ta));
    std::memset(&tb, 0, sizeof(tb));
    if (both_f8) {
      p.a = a;  // the staging warps read both operands
      p.wq = static_cast<const uint8_t*>(w);
      set_kernel_family(1);
      if (tile_m == 64) return launch_fp8<1>(a_dtype, w_dtype, ta, tb, p, st);
      return launch_fp8<2>(a_dtype, w_dtype, ta, tb, p, st);
    }
    rc = make_tmap_2d(&ta, a, DT_U8, m, k, tile_m);
    if (rc != OK) return rc;
    rc = make_tmap_2d(&tb, w, DT_U8, n, k, bn);
    if (rc != OK) return rc;
    set_kernel_family(1);
    {
      if (tile_m == 64) return bn == 256 ? launch_int8<1, 256>(ta, tb, p, st) : launch_int8<1, 128>(ta, tb, p, st);
      return bn == 256 ? launch_int8<2, 256>(ta, tb, p, st) : launch_int8<2, 128>(ta, tb, p, st);
    }
  }
  if (q_dt != 0)
    return fail(ERR_UNSUPPORTED, "qbytes_mm_quantized: needs int8 x int8 or fp8 x fp8 operands, K %% 16 == 0 and "
                                 "16-byte aligned buffers");
  // weight-only 8-bit: fp16 / bf16 activations x int8 / fp8 weights, converted in-kernel (reference rounding order)
  const bool a_half = (a_dtype == DT_F16 || a_dtype == DT_BF16);
  if (a_half && out_dtype == a_dtype && (k % 16 == 0) && reinterpret_cast<uintptr_t>(a) % 16 == 0 &&
      reinterpret_cast<uintptr_t>(w) % 16 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0 && route != ROUTE_QBYTES_SIMT) {
    constexpr int BN = 128;
    GemmParams p = base_params();
    p.scales = nullptr;  // applied to the weights before the MMA, like the reference does
    p.wq = static_cast<const uint8_t*>(w);
    p.wscale = scales;
    p.w_dt = w_dtype;
    p.num_n_blocks = static_cast<int>((n + BN - 1) / BN);
    p.num_m_blocks = static_cast<int>((m + tile_m - 1) / tile_m);
    CUtensorMap ta, tb;
    std::memset(&tb, 0, sizeof(tb));
    rc = make_tmap_2d(&ta, a, a_dtype, m, k, tile_m);
    if (rc != OK) return rc;
    set_kernel_family(1);
#define QB_LAUNCH_BYTES(KIND, WT, WK)                                                                   \
  (tile_m == 128 ? launch_gemm<GemmCfg<KIND, BSrc::BYTES, 2, BN, WT, false, WK>>(ta, tb, p, st)         \
                 : launch_gemm<GemmCfg<KIND, BSrc::BYTES, 1, BN, WT, false, WK>>(ta, tb, p, st))
    const int wk = (w_dtype == DT_I8) ? 0 : (w_dtype == DT_E4M3 ? 1 : (w_dtype == DT_E5M2 ? 2 : 3));
    if (a_dtype == DT_BF16) {
      if (wk == 0) return QB_LAUNCH_BYTES(MmaKind::BF16, __nv_bfloat16, 0);
      if (wk == 1) return QB_LAUNCH_BYTES(MmaKind::BF16, __nv_bfloat16, 1);
      if (wk == 2) return QB_LAUNCH_BYTES(MmaKind::BF16, __nv_bfloat16, 2);
      return QB_LAUNCH_BYTES(MmaKind::BF16, __nv_bfloat16, 3);
    }
    if (wk == 0) return QB_LAUNCH_BYTES(MmaKind::F16, __half, 0);
    if (wk == 1) return QB_LAUNCH_BYTES(MmaKind::F16, __half, 1);
    if (wk == 2) return QB_LAUNCH_BYTES(MmaKind::F16, __half, 2);
    return QB_LAUNCH_BYTES(MmaKind::F16, __half, 3);
#undef QB_LAUNCH_BYTES
  }
  set_kernel_family(2);
  rc = launch_qbytes_mm_simt(a, w, scales, bias, out, static_cast<int>(m), static_cast<int>(n), static_cast<int>(k),
                             a_dtype, w_dtype, out_dtype, st);
  return rc == OK ? OK : fail(rc, "qbytes_mm: CUDA-core kernel launch failed");
}

}  // namespace qb

using namespace qb;

extern "C" {

int qb200_qbytes_mm(const void* a, const void* w, const void* scales, const void* bias, void* out, int64_t m,
                    int64_t n, int64_t k, int a_dtype, int w_dtype, int out_dtype, void* stream) {
  return qbytes_mm_impl(a, w, scales, bias, out, m, n, k, a_dtype, w_dtype, out_dtype, 0, nullptr, stream);
}

int qb200_qbytes_mm_quantized(const void* a, const void* w, const void* scales, const void* bias, void* out_q,
                              const void* out_scale, int64_t m, int64_t n, int64_t k, int a_dtype, int w_dtype,
                              int scale_dtype, int q_dtype, void* stream) {
  if (q_dtype != DT_I8 && q_dtype != DT_E4M3 && q_dtype != DT_E5M2)
    return fail(ERR_ARG, "qbytes_mm_quantized: unsupported target dtype %d", q_dtype);
  if (scales == nullptr || out_scale == nullptr) return fail(ERR_ARG, "qbytes_mm_quantized: scales / out_scale missing");
  return qbytes_mm_impl(a, w, scales, bias, out_q, m, n, k, a_dtype, w_dtype, scale_dtype, q_dtype, out_scale, stream);
}

}  // extern "C"
