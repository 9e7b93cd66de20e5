// qb200_qbits_mm_grad_input / qb200_qbytes_mm_grad_input: argument checks and the instantiations of the input-gradient
// kernel (gemm_tc_dgrad.cuh) of the packed-int4 and 8-bit linears.
#include "../../include/quanto_b200.h"

#include "gemm_tc_dgrad.cuh"
#include "host_common.cuh"

namespace qb {

template <class Cfg>
static int launch_dgrad(const CUtensorMap& tg, const DgradParams& p, cudaStream_t stream) {
  return launch_persistent<gemm_dgrad_kernel<Cfg>, typename Cfg::Pipe>(p.num_m_blocks * p.num_k_blocks, stream,
                                                                       "gemm_dgrad_kernel launch", tg, p);
}

// The autograd engine runs a CUDA backward on a thread of its own, where no context may be current yet: the driver's
// tensor-map encoder (unlike the runtime calls) then fails with CUDA_ERROR_INVALID_CONTEXT.  cudaSetDevice makes the
// device's primary context current on the calling thread.
static int make_context_current() { return check_cuda(cudaSetDevice(current_device()), "cudaSetDevice"); }

static int qbits_grad_input_impl(const void* grad_out, const uint8_t* packed, const void* scale, const void* shift,
                                 void* grad_in, int64_t m, int64_t n, int64_t k, int group, int dtype, int shift_is_int,
                                 cudaStream_t stream) {
  set_kernel_family(0);
  if (m < 0 || n <= 0 || k <= 0 || group <= 0) return fail(ERR_ARG, "qbits_mm_grad_input: bad shape");
  if (!is_float_dtype(dtype)) return fail(ERR_ARG, "qbits_mm_grad_input: dtype must be f32, f16 or bf16");
  if (k % group != 0) return fail(ERR_ARG, "qbits_mm_grad_input: group %d does not divide K = %lld", group, (long long)k);
  if (m > INT32_MAX || n > INT32_MAX || k > INT32_MAX) return fail(ERR_UNSUPPORTED, "qbits_mm_grad_input: dimension too large");
  if (dtype == DT_F32) return fail(ERR_UNSUPPORTED, "qbits_mm_grad_input: the kernel takes f16 / bf16 gradients");
  if (n % 16 != 0 || k % 16 != 0 || !(group == 32 || group % 64 == 0))
    return fail(ERR_UNSUPPORTED, "qbits_mm_grad_input: needs N %% 16 == 0, K %% 16 == 0 and group 32 or a multiple of 64");
  if (!aligned16(grad_out) || !aligned16(packed) || !aligned16(grad_in))
    return fail(ERR_UNSUPPORTED, "qbits_mm_grad_input: grad_out, packed and grad_in must be 16-byte aligned");
  if (m == 0) return OK;
  int rc = check_arch("qbits_mm_grad_input");
  if (rc == OK) rc = make_context_current();
  if (rc != OK) return rc;

  DgradParams p{};
  p.out = grad_in;
  p.w = packed;
  p.wscale = scale;
  p.wshift = shift;
  p.M = static_cast<int>(m);
  p.N = static_cast<int>(n);
  p.K = static_cast<int>(k);
  p.group = group;
  p.group_log2 = group_log2(group);
  const int tile_m = wgmma_tile_m(m);
  p.num_m_blocks = static_cast<int>((m + tile_m - 1) / tile_m);
  p.num_k_blocks = static_cast<int>((k + 127) / 128);
  p.red_blocks = static_cast<int>((n / 2 + 63) / 64);
  CUtensorMap tg;
  rc = make_tmap_planes(&tg, grad_out, dtype, m, n, tile_m);
  if (rc != OK) return rc;
  set_kernel_family(1);
  return dispatch_act16_zp(dtype, shift_is_int, [&](auto act, auto ZP) {
    return dispatch_mwg(tile_m, [&](auto MWG) {
      return launch_dgrad<DgradCfg<true, MWG, typename decltype(act)::WT, ZP>>(tg, p, stream);
    });
  });
}

static int qbytes_grad_input_impl(const void* grad_out, const void* w, const void* scales, void* grad_in, int64_t m,
                                  int64_t n, int64_t k, int w_dtype, int dtype, cudaStream_t stream) {
  set_kernel_family(0);
  if (m < 0 || n <= 0 || k <= 0) return fail(ERR_ARG, "qbytes_mm_grad_input: bad shape");
  if (!is_code_dtype(w_dtype)) return fail(ERR_ARG, "qbytes_mm_grad_input: weights must be int8 or float8");
  if (!is_float_dtype(dtype)) return fail(ERR_ARG, "qbytes_mm_grad_input: dtype must be f32, f16 or bf16");
  if (m > INT32_MAX || n > INT32_MAX || k > INT32_MAX) return fail(ERR_UNSUPPORTED, "qbytes_mm_grad_input: dimension too large");
  if (dtype == DT_F32) return fail(ERR_UNSUPPORTED, "qbytes_mm_grad_input: the kernel takes f16 / bf16 gradients");
  if (n % 8 != 0 || k % 16 != 0) return fail(ERR_UNSUPPORTED, "qbytes_mm_grad_input: needs N %% 8 == 0 and K %% 16 == 0");
  if (!aligned16(grad_out) || !aligned16(w) || !aligned16(grad_in))
    return fail(ERR_UNSUPPORTED, "qbytes_mm_grad_input: grad_out, w and grad_in must be 16-byte aligned");
  if (m == 0) return OK;
  int rc = check_arch("qbytes_mm_grad_input");
  if (rc == OK) rc = make_context_current();
  if (rc != OK) return rc;

  DgradParams p{};
  p.out = grad_in;
  p.w = static_cast<const uint8_t*>(w);
  p.wscale = scales;
  p.M = static_cast<int>(m);
  p.N = static_cast<int>(n);
  p.K = static_cast<int>(k);
  const int tile_m = wgmma_tile_m(m);
  p.num_m_blocks = static_cast<int>((m + tile_m - 1) / tile_m);
  p.num_k_blocks = static_cast<int>((k + 127) / 128);
  p.red_blocks = static_cast<int>((n + 63) / 64);
  CUtensorMap tg;
  rc = make_tmap_2d(&tg, grad_out, dtype, m, n, tile_m);
  if (rc != OK) return rc;
  set_kernel_family(1);
  return dispatch_act16(dtype, [&](auto act) {
    return dispatch_wkind(w_dtype, [&](auto WK) {
      return dispatch_mwg(tile_m, [&](auto MWG) {
        return launch_dgrad<DgradCfg<false, MWG, typename decltype(act)::WT, false, WK>>(tg, p, stream);
      });
    });
  });
}

}  // namespace qb

using namespace qb;

extern "C" {

int qb200_qbits_mm_grad_input(const void* grad_out, const uint8_t* packed, const void* scale, const void* shift,
                              void* grad_in, int64_t m, int64_t n, int64_t k, int group, int dtype, int shift_is_int,
                              void* stream) {
  return qbits_grad_input_impl(grad_out, packed, scale, shift, grad_in, m, n, k, group, dtype, shift_is_int,
                               static_cast<cudaStream_t>(stream));
}

int qb200_qbytes_mm_grad_input(const void* grad_out, const void* w, const void* scales, void* grad_in, int64_t m,
                               int64_t n, int64_t k, int w_dtype, int dtype, void* stream) {
  return qbytes_grad_input_impl(grad_out, w, scales, grad_in, m, n, k, w_dtype, dtype, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
