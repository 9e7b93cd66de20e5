// qb200_qbits_conv2d / qb200_qbytes_conv2d: argument checks, tile choice and the instantiations of the implicit-GEMM
// convolution (conv_tc.cuh).
#include "../../include/quanto_b200.h"

#include "conv_tc.cuh"
#include "host_common.cuh"

namespace qb {

struct ConvArgs {
  const void* x;
  const void* bias;
  void* out;
  int64_t batch, cin, h, w, cout, kh, kw;
  int sh, sw, ph, pw, dh, dw;
  int dtype;
  cudaStream_t stream;
};

template <class G>
static int launch_conv(const GemmParams& p, const ConvGeom& g, cudaStream_t st) {
  using C = ConvCfg<G>;
  return launch_persistent<conv_tc_kernel<C>, typename C::Pipe>(p.num_m_blocks * p.num_n_blocks, st,
                                                                "conv_tc_kernel launch", p, g);
}

// Shape checks shared by both entry points; fills the GEMM view (M, N, K) and the geometry.  Offsets into the input
// and output are 64-bit in the kernel: only M, N, K and the spatial sizes must fit in int32.
static int conv_setup(const char* what, const ConvArgs& a, GemmParams* p, ConvGeom* g) {
  if (a.batch < 0 || a.cin <= 0 || a.h <= 0 || a.w <= 0 || a.cout <= 0 || a.kh <= 0 || a.kw <= 0)
    return fail(ERR_ARG, "%s: bad shape", what);
  if (a.sh < 1 || a.sw < 1 || a.dh < 1 || a.dw < 1 || a.ph < 0 || a.pw < 0)
    return fail(ERR_ARG, "%s: stride and dilation must be >= 1, padding >= 0", what);
  if (a.dtype != DT_BF16 && a.dtype != DT_F16) return fail(ERR_UNSUPPORTED, "%s: bf16 / fp16 activations only", what);
  const int64_t ho = (a.h + 2 * a.ph - a.dh * (a.kh - 1) - 1) / a.sh + 1;
  const int64_t wo = (a.w + 2 * a.pw - a.dw * (a.kw - 1) - 1) / a.sw + 1;
  if (a.h + 2 * a.ph < a.dh * (a.kh - 1) + 1 || a.w + 2 * a.pw < a.dw * (a.kw - 1) + 1 || ho <= 0 || wo <= 0)
    return fail(ERR_ARG, "%s: the kernel is larger than the padded input", what);
  const int64_t m = a.batch * ho * wo, k = a.cin * a.kh * a.kw;
  if (m > INT32_MAX || k > INT32_MAX || a.cout > INT32_MAX || a.h > INT32_MAX / 2 || a.w > INT32_MAX / 2)
    return fail(ERR_UNSUPPORTED, "%s: dimension too large", what);
  if (k % 16 != 0) return fail(ERR_UNSUPPORTED, "%s: Cin * kh * kw = %lld is not a multiple of 16", what, (long long)k);
  if (reinterpret_cast<uintptr_t>(a.x) % 2 != 0 || reinterpret_cast<uintptr_t>(a.out) % 2 != 0 ||
      reinterpret_cast<uintptr_t>(a.bias) % 2 != 0)
    return fail(ERR_UNSUPPORTED, "%s: input, bias and output must be aligned to their elements", what);
  *p = dense_gemm_params(a.out, a.bias, a.dtype, m, a.cout, k);
  p->dbg = debug_flags();
  *g = ConvGeom{a.x, static_cast<int>(a.cin), static_cast<int>(a.h), static_cast<int>(a.w), static_cast<int>(ho),
                static_cast<int>(wo), static_cast<int>(a.kh), static_cast<int>(a.kw), a.sh, a.sw, a.ph, a.pw, a.dh, a.dw};
  return OK;
}

// Rows per M tile: 64 when the 128-row tiles would leave SMs idle (a small batch or feature map), else 128; test
// override OVR_CONV_TILE_M forces either.  Sets the tile counts; n_tiles = N tiles (128 out-features each).
static int conv_tile_m(GemmParams* p, int64_t n_tiles) {
  int t = (((p->M + 127) / 128) * n_tiles < current_sm_count()) ? 64 : 128;
  const int force = test_override(OVR_CONV_TILE_M);
  if (force == 64 || force == 128) t = force;
  p->num_m_blocks = (p->M + t - 1) / t;
  p->num_n_blocks = static_cast<int>(n_tiles);
  return t;
}

}  // namespace qb

using namespace qb;

extern "C" {

int qb200_qbits_conv2d(const void* x, const uint8_t* packed, const void* scale, const void* shift, const void* bias,
                       void* out, int64_t batch, int64_t cin, int64_t h, int64_t w, int64_t cout, int64_t kh, int64_t kw,
                       int stride_h, int stride_w, int pad_h, int pad_w, int dil_h, int dil_w, int group, int bits,
                       int dtype, int shift_is_int, void* stream) {
  set_kernel_family(0);
  const ConvArgs a{x, bias, out, batch, cin, h, w, cout, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, dtype,
                   static_cast<cudaStream_t>(stream)};
  GemmParams p;
  ConvGeom g;
  int rc = conv_setup("qbits_conv2d", a, &p, &g);
  if (rc != OK) return rc;
  if (group <= 0 || p.K % group != 0) return fail(ERR_ARG, "qbits_conv2d: group %d does not divide K = %d", group, p.K);
  if (bits != 4) return fail(ERR_UNSUPPORTED, "qbits_conv2d: 4-bit weights only (got %d)", bits);
  if (cout % 2 != 0) return fail(ERR_UNSUPPORTED, "qbits_conv2d: odd Cout");
  // a 32-k half of a stage must lie inside one group (conv_tc.cuh); one group per row (per-axis) always does
  if (group % 32 != 0 && group != p.K)
    return fail(ERR_UNSUPPORTED, "qbits_conv2d: group %d is neither a multiple of 32 nor K", group);
  if (!aligned16(packed)) return fail(ERR_UNSUPPORTED, "qbits_conv2d: packed weights not 16-byte aligned");
  if (p.M == 0) return OK;
  rc = check_arch("qbits_conv2d");
  if (rc != OK) return rc;
  p.wq = packed;
  p.wscale = scale;
  p.wshift = shift;
  p.group = group;
  p.group_log2 = group_log2(group);
  p.shift_is_int = shift_is_int;
  const int t = conv_tile_m(&p, (cout / 2 + 63) / 64);
  set_kernel_family(5);
  return dispatch_act16_zp(dtype, shift_is_int, [&](auto act, auto ZP) {
    return dispatch_mwg(t, [&](auto MWG) {
      using A = decltype(act);
      return launch_conv<GemmCfg<A::KIND, BSrc::INT4, MWG, 128, typename A::WT, ZP>>(p, g, a.stream);
    });
  });
}

int qb200_qbytes_conv2d(const void* x, const void* wq, const void* scales, const void* bias, void* out, int64_t batch,
                        int64_t cin, int64_t h, int64_t w, int64_t cout, int64_t kh, int64_t kw, int stride_h,
                        int stride_w, int pad_h, int pad_w, int dil_h, int dil_w, int w_dtype, int dtype, void* stream) {
  set_kernel_family(0);
  if (!is_code_dtype(w_dtype)) return fail(ERR_ARG, "qbytes_conv2d: weights must be int8 or float8");
  const ConvArgs a{x, bias, out, batch, cin, h, w, cout, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, dtype,
                   static_cast<cudaStream_t>(stream)};
  GemmParams p;
  ConvGeom g;
  int rc = conv_setup("qbytes_conv2d", a, &p, &g);
  if (rc != OK) return rc;
  if (!aligned16(wq)) return fail(ERR_UNSUPPORTED, "qbytes_conv2d: weights not 16-byte aligned");
  if (p.M == 0) return OK;
  rc = check_arch("qbytes_conv2d");
  if (rc != OK) return rc;
  p.wq = static_cast<const uint8_t*>(wq);
  p.wscale = scales;
  p.w_dt = w_dtype;
  const int t = conv_tile_m(&p, (cout + 127) / 128);
  set_kernel_family(5);
  return dispatch_act16(dtype, [&](auto act) {
    return dispatch_wkind(w_dtype, [&](auto WK) {
      return dispatch_mwg(t, [&](auto MWG) {
        using A = decltype(act);
        return launch_conv<GemmCfg<A::KIND, BSrc::BYTES, MWG, 128, typename A::WT, false, WK>>(p, g, a.stream);
      });
    });
  });
}

}  // extern "C"
