// qb200_qbytes_mm / qb200_qbytes_mm_quantized: argument checks, kernel selection and the instantiations of the 8-bit
// paths: int8 x int8 on wgmma with both operands fed by TMA (gemm_tc.cuh), fp8 x fp8 and weight-only fp16 / bf16 x
// int8 / fp8 with the conversion to 16 bits in the staging warps, and the shape-agnostic CUDA-core kernel.
#include "../../include/quanto_b200.h"

#include "gemm_tc.cuh"
#include "host_common.cuh"

namespace qb {

int launch_qbytes_mm_simt(const void*, const void*, const void*, const void*, void*, int, int, int, int, int, int,
                          cudaStream_t);

// Columns of tensor-core work per SM for a tile of BM x bn: waves x bn (wave quantisation included).
static int64_t wave_cost(int64_t m, int64_t n, int bm, int bn) {
  const int64_t tiles = ((m + bm - 1) / bm) * ((n + bn - 1) / bn);
  const int64_t sms = current_sm_count();
  return ((tiles + sms - 1) / sms) * bn;
}

// fp8 x fp8: both operands converted to bf16 by the staging warps (exact), bf16 MMAs with fp32 accumulation.  Hopper's
// native fp8 MMA accumulates with fewer bits than fp32 and misses the exact-product / fp32-sum contract.  Shipped for
// the e4m3 / e5m2 pairs (WKIND, AKIND: 1 e4m3, 2 e5m2) with bf16 staging only.
template <int MWG, int WK, int AK>
using F8Cfg = GemmCfg<MmaKind::BF16, BSrc::F8, MWG, 128, __nv_bfloat16, false, WK, AK>;

// q_dt != 0: the output is quantised in the epilogue (out = [M, N] bytes, q_scale = device pointer to the per-tensor
// output scale in out_dtype); only the int8 x int8 / fp8 x fp8 tensor-core kernels do that.
static int qbytes_mm_impl(const void* a, const void* w, const void* scales, const void* bias, void* out, int64_t m,
                          int64_t n, int64_t k, int a_dtype, int w_dtype, int out_dtype, int q_dt, const void* q_scale,
                          void* stream) {
  set_kernel_family(0);
  if (m < 0 || n <= 0 || k <= 0) return fail(ERR_ARG, "qbytes_mm: bad shape");
  if (!is_float_dtype(out_dtype)) return fail(ERR_ARG, "qbytes_mm: scales/out dtype must be floating point");
  if (!is_code_dtype(w_dtype)) return fail(ERR_ARG, "qbytes_mm: weights must be int8 or float8");
  if (a_dtype < DT_F32 || a_dtype > DT_E4M3FNUZ || a_dtype == DT_U8) return fail(ERR_ARG, "qbytes_mm: bad activation dtype");
  if (m > INT32_MAX || n > INT32_MAX || k > INT32_MAX) return fail(ERR_UNSUPPORTED, "qbytes_mm: dimension too large");
  if (m == 0) return OK;
  int rc = check_arch("qbytes_mm");
  if (rc != OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int route = test_override(OVR_QBYTES_ROUTE);

  const int tile_m = wgmma_tile_m(m);

  const bool both_i8 = (a_dtype == DT_I8 && w_dtype == DT_I8);
  const bool both_f8 = ((a_dtype == DT_E4M3 || a_dtype == DT_E5M2) && (w_dtype == DT_E4M3 || w_dtype == DT_E5M2));
  const bool tma_ok = (k % 16 == 0) && aligned16(a) && aligned16(w) && aligned16(out);
  if ((both_i8 || both_f8) && tma_ok && route != ROUTE_QBYTES_SIMT) {
    GemmParams p = dense_gemm_params(out, bias, out_dtype, m, n, k);
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
    if (both_f8) {
      p.a = a;  // the staging warps read both operands
      p.wq = static_cast<const uint8_t*>(w);
      set_kernel_family(1);
      return dispatch_mwg(tile_m, [&](auto MWG) {
        constexpr int E4 = 1, E5 = 2;
        if (a_dtype == DT_E4M3 && w_dtype == DT_E4M3) return launch_gemm_tc<F8Cfg<MWG, E4, E4>>(nullptr, nullptr, nullptr, p, st);
        if (a_dtype == DT_E4M3) return launch_gemm_tc<F8Cfg<MWG, E5, E4>>(nullptr, nullptr, nullptr, p, st);
        if (w_dtype == DT_E4M3) return launch_gemm_tc<F8Cfg<MWG, E4, E5>>(nullptr, nullptr, nullptr, p, st);
        return launch_gemm_tc<F8Cfg<MWG, E5, E5>>(nullptr, nullptr, nullptr, p, st);
      });
    }
    CUtensorMap ta, tb;
    rc = make_tmap_2d(&ta, a, DT_U8, m, k, tile_m);
    if (rc != OK) return rc;
    rc = make_tmap_2d(&tb, w, DT_U8, n, k, bn);
    if (rc != OK) return rc;
    set_kernel_family(1);
    return dispatch_mwg(tile_m, [&](auto MWG) {
      if (bn == 256) return launch_gemm_tc<GemmCfg<MmaKind::I8, BSrc::TMA, MWG, 256>>(&ta, &tb, nullptr, p, st);
      return launch_gemm_tc<GemmCfg<MmaKind::I8, BSrc::TMA, MWG, 128>>(&ta, &tb, nullptr, p, st);
    });
  }
  if (q_dt != 0)
    return fail(ERR_UNSUPPORTED, "qbytes_mm_quantized: needs int8 x int8 or fp8 x fp8 operands, K %% 16 == 0 and "
                                 "16-byte aligned buffers");
  // weight-only 8-bit: fp16 / bf16 activations x int8 / fp8 weights, converted in-kernel (reference rounding order)
  const bool a_half = (a_dtype == DT_F16 || a_dtype == DT_BF16);
  if (a_half && out_dtype == a_dtype && (k % 16 == 0) && aligned16(a) && aligned16(w) && aligned16(out) &&
      route != ROUTE_QBYTES_SIMT) {
    constexpr int BN = 128;
    GemmParams p = dense_gemm_params(out, bias, out_dtype, m, n, k);
    p.scales = nullptr;  // applied to the weights before the MMA, like the reference does
    p.wq = static_cast<const uint8_t*>(w);
    p.wscale = scales;
    p.w_dt = w_dtype;
    p.num_n_blocks = static_cast<int>((n + BN - 1) / BN);
    p.num_m_blocks = static_cast<int>((m + tile_m - 1) / tile_m);
    CUtensorMap ta;
    rc = make_tmap_2d(&ta, a, a_dtype, m, k, tile_m);
    if (rc != OK) return rc;
    set_kernel_family(1);
    return dispatch_act16(a_dtype, [&](auto act) {
      return dispatch_wkind(w_dtype, [&](auto WK) {
        return dispatch_mwg(tile_m, [&](auto MWG) {
          using A = decltype(act);
          return launch_gemm_tc<GemmCfg<A::KIND, BSrc::BYTES, MWG, BN, typename A::WT, false, WK>>(&ta, nullptr, nullptr,
                                                                                                   p, st);
        });
      });
    });
  }
  set_kernel_family(2);
  return launch_qbytes_mm_simt(a, w, scales, bias, out, static_cast<int>(m), static_cast<int>(n), static_cast<int>(k),
                               a_dtype, w_dtype, out_dtype, st);
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
  // no float8_e4m3fnuz output: the fused epilogue quantises to int8, e4m3fn and e5m2 only
  if (!is_code_dtype(q_dtype) || q_dtype == DT_E4M3FNUZ)
    return fail(ERR_ARG, "qbytes_mm_quantized: unsupported target dtype %d", q_dtype);
  if (scales == nullptr || out_scale == nullptr) return fail(ERR_ARG, "qbytes_mm_quantized: scales / out_scale missing");
  return qbytes_mm_impl(a, w, scales, bias, out_q, m, n, k, a_dtype, w_dtype, scale_dtype, q_dtype, out_scale, stream);
}

}  // extern "C"
