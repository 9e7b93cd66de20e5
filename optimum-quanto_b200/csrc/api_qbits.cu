// qb200_qbits_mm / qb200_qbits_mm_gather: argument checks, kernel selection and the wgmma instantiations of the fused
// packed-int4 linear (gemm_tc.cuh).  The small-M gemv kernels live in api_qbits_small.cu.
#include "../../include/quanto_b200.h"

#include <cstring>

#include "api_qbits.cuh"
#include "gemm_tc.cuh"

namespace qb {

int launch_qbits_mm_simt(const void*, const uint8_t*, const void*, const void*, const void*, void*, int, int, int, int,
                         int, int, int, int64_t, int64_t, cudaStream_t);

template <class C>
static int launch_gemm_w4(const CUtensorMap& ta, const CUtensorMap& tw, const CUtensorMap& tout, const GemmParams& p,
                          cudaStream_t st) {
  return launch_persistent<gemm_w4_kernel<C>, C>(p.num_m_blocks * p.num_n_blocks, st, "gemm_w4_kernel launch", ta, tw,
                                                 tout, p);
}

// Which int4 wgmma kernel runs a problem of m_blocks 128-token blocks and half_n packed rows.  The swap-AB kernel
// (gemm_w4_kernel) was measured on tiles of 128 tokens x 128 packed rows, the same MACs as its 256 x 64 tiles: such a
// tile took about 1.8x the time the weight-staging kernel (gemm_tc_kernel) takes for its 128 x 64 tile (H100 SXM, bf16,
// M = 4096: 1.10 vs 1.22 ms for twice the tiles), so it wins once its tiles fill every SM and its waves, 1.8x as long,
// are fewer than 5/9 of the staging kernel's.  At N = 14336 on 132 SMs that is M = 512, 768 and M >= 1536; small batches
// (M <= 256) and M = 1024, 1280 keep the staging kernel.
static bool use_swap_kernel(int64_t m_blocks, int64_t half_n) {
  const int64_t sms = current_sm_count();
  const int64_t tiles_swap = m_blocks * ((half_n + 127) / 128), tiles_staged = m_blocks * ((half_n + 63) / 64);
  if (tiles_swap < sms) return false;
  return 9 * ((tiles_swap + sms - 1) / sms) < 5 * ((tiles_staged + sms - 1) / sms);
}

// Token rows per tile of the swap-AB kernel: 64 while M <= 64; else 256 where the 256 x 64 tiles cost less than the
// 128 x 128 ones, else 128.  Both tile sizes cover the same packed rows per token, so the costs compare as the tokens
// the tiles span (M rounded up to the tile) times the time per token row: 0.72-0.77 as much at T = 256 (H100 SXM, bf16,
// N = 14336, K = 4096: 0.755 vs 0.980 ms at M = 4096, 0.111 vs 0.151 at M = 512, 0.408 vs 0.566 at M = 2048), taken
// as 3/4.  So M <= 128 keeps 128-token tiles (a 256-token tile would be more than half empty), and so does a ragged
// M = 256 j + r with 0 < r <= 128 while j is small (M = 257 ... 384: 512 tokens against 384).  use_swap_kernel counts
// 128 x 128 tiles: the tile chosen here is, by this estimate, no slower than those.  Test override OVR_TILE_M forces 64,
// 128 or 256.
static int swap_tile_t(int64_t m) {
  const int force = test_override(OVR_TILE_M);
  if (force == 64 || force == 128 || force == 256) return force;
  if (m <= 64) return 64;
  const int64_t span256 = (m + 255) / 256 * 256, span128 = (m + 127) / 128 * 128;
  return 3 * span256 < 4 * span128 ? 256 : 128;
}

static int qbits_mm_impl(QbitsArgs& q) {
  set_kernel_family(0);
  const int64_t m = q.m, n = q.n, k = q.k;
  const int group = q.group, dtype = q.dtype;
  if (m < 0 || n <= 0 || k <= 0 || group <= 0) return fail(ERR_ARG, "qbits_mm: bad shape");
  if (!is_float_dtype(dtype)) return fail(ERR_ARG, "qbits_mm: dtype must be f32, f16 or bf16");
  if (q.bits != 4 && q.bits != 2) return fail(ERR_ARG, "qbits_mm: bits must be 2 or 4 (got %d)", q.bits);
  if (k % group != 0) return fail(ERR_ARG, "qbits_mm: group %d does not divide K = %lld", group, (long long)k);
  if (m > INT32_MAX || n > INT32_MAX || k > INT32_MAX || q.ld > INT32_MAX) return fail(ERR_UNSUPPORTED, "qbits_mm: dimension too large");
  if (m == 0) return OK;
  int rc = check_arch("qbits_mm");
  if (rc != OK) return rc;
  const bool gathered = q.g.n_out > 1;
  // tensor-core kernels: 4-bit, 16-bit activations, N even, K % 16 == 0, group 32 or a multiple of 64, aligned buffers.
  // Everything else runs on the shape-agnostic CUDA-core kernel (same operands, same rounding order).
  const bool tc_ok = q.bits == 4 && (dtype == DT_BF16 || dtype == DT_F16) && n % 2 == 0 && k % 16 == 0 &&
                     (group == 32 || group % 64 == 0) && aligned16(q.packed) && aligned16(q.out) && aligned16(q.a);
  if (!tc_ok) {
    if (gathered) return fail(ERR_UNSUPPORTED, "qbits_mm_gather: the fused gather exists for the tensor-core kernels only");
    set_kernel_family(2);
    return launch_qbits_mm_simt(q.a, q.packed, q.scale, q.shift, q.bias, q.out, static_cast<int>(m), static_cast<int>(n),
                                static_cast<int>(k), group, q.bits, dtype, q.shift_is_int, q.ld, q.col0, q.stream);
  }
  q.group_log2 = group_log2(group);

  bool handled = false;
  rc = qbits_small_dispatch(q, &handled);
  if (rc != OK || handled) return rc;

  GemmParams p = dense_gemm_params(q.out, q.bias, dtype, m, n, k);
  p.g = q.g;  // the fused gather's peer buffers and column slab
  p.ld = static_cast<int>(q.ld);
  p.col0 = static_cast<int>(q.col0);
  p.wq = q.packed;
  p.wscale = q.scale;
  p.wshift = q.shift;
  p.group = group;
  p.group_log2 = q.group_log2;
  p.shift_is_int = q.shift_is_int;
  p.dbg = debug_flags();
  const int tile_m = wgmma_tile_m(m);
  const int64_t half_n = n / 2;
  // OVR_TILE_M = 256 names the swap-AB kernel's 256-token tile, at any shape
  const bool swap = test_override(OVR_TILE_M) == 256 || use_swap_kernel((m + tile_m - 1) / tile_m, half_n);
  // tile: t tokens x pr packed rows (swap-AB: both nibble planes of each; 64 and 128 tokens go with 128 packed rows,
  // 256 tokens with 64) or x 64 packed rows (weight staging)
  const int t = swap ? swap_tile_t(m) : tile_m;
  const int pr = (swap && t != 256) ? 128 : 64;
  const int64_t m_blocks = (m + t - 1) / t;
  p.num_m_blocks = static_cast<int>(m_blocks);
  p.num_n_blocks = static_cast<int>((half_n + pr - 1) / pr);
  CUtensorMap ta, tw;
  rc = make_tmap_2d(&ta, q.a, dtype, m, k, t);
  if (rc != OK) return rc;
  if (swap) {
    rc = make_tmap_packed(&tw, q.packed, half_n, k, pr);
    if (rc != OK) return rc;
  }
  // The epilogue stores each warpgroup's tile with TMA when the output is one dense, 16-byte aligned [M, N] buffer whose
  // two nibble planes [M, 2, N/2] have 16-byte aligned rows (N % 16 == 0).  Everything else -- the fused gather's peer
  // buffers and column slab, N % 16 != 0, a map the driver declines -- stores with ordinary stores.
  CUtensorMap tout;
  std::memset(&tout, 0, sizeof(tout));
  p.epi_tma = 0;
  if (test_override(OVR_INT4_EPILOGUE) != 1 && q.g.n_out == 1 && q.g.out_peer[0] == q.out && q.ld == n && q.col0 == 0 &&
      n % 16 == 0 && aligned16(q.out)) {
    if (make_tmap_planes(&tout, q.out, dtype, m, n, swap ? t : 64) == OK) p.epi_tma = 1;
    else std::memset(&tout, 0, sizeof(tout));
  }
  set_kernel_family(1);
  return dispatch_act16_zp(dtype, q.shift_is_int, [&](auto act, auto ZP) {
    using A = decltype(act);
    if (!swap)
      return dispatch_mwg(tile_m, [&](auto MWG) {
        return launch_gemm_tc<GemmCfg<A::KIND, BSrc::INT4, MWG, 128, typename A::WT, ZP>>(&ta, nullptr, &tout, p,
                                                                                          q.stream);
      });
    if (t == 64) return launch_gemm_w4<W4Cfg<A::KIND, 64, typename A::WT, ZP>>(ta, tw, tout, p, q.stream);
    if (t == 128) return launch_gemm_w4<W4Cfg<A::KIND, 128, typename A::WT, ZP>>(ta, tw, tout, p, q.stream);
    return launch_gemm_w4<W4Cfg<A::KIND, 256, typename A::WT, ZP>>(ta, tw, tout, p, q.stream);
  });
}

}  // namespace qb

using namespace qb;

extern "C" {

int64_t qb200_qbits_mm_workspace_bytes(int64_t m, int64_t n, int64_t k) { return qbits_small_workspace_bytes(m, n, k); }

int qb200_qbits_ring_plan(int64_t m, int64_t n, int64_t k, int group, int zeropoint, int grid, int* out5) {
  if (out5 == nullptr) return 0;
  return qbits_ring_plan(m, n, k, group, zeropoint, grid, out5);
}

int qb200_qbits_mm(const void* a, const uint8_t* packed, const void* scale, const void* shift, const void* bias,
                   void* out, int64_t m, int64_t n, int64_t k, int group, int bits, int dtype, int shift_is_int,
                   void* workspace, int64_t workspace_bytes, void* stream) {
  QbitsArgs q{};
  q.a = a; q.packed = packed; q.scale = scale; q.shift = shift; q.bias = bias; q.out = out;
  q.m = m; q.n = n; q.k = k; q.ld = n; q.col0 = 0;
  q.group = group; q.bits = bits; q.dtype = dtype; q.shift_is_int = shift_is_int;
  q.workspace = workspace; q.workspace_bytes = workspace_bytes;
  q.g.out_peer[0] = out;
  q.g.n_out = 1;
  q.g.world = 1;
  q.stream = static_cast<cudaStream_t>(stream);
  return qbits_mm_impl(q);
}

int qb200_qbits_mm_gather(const void* a, const uint8_t* packed, const void* scale, const void* shift, const void* bias,
                          void* const* out_peers, void* const* flag_peers, int world, int rank, int wait_flags,
                          int64_t m, int64_t n_local, int64_t k, int group, int dtype, int shift_is_int, void* workspace,
                          int64_t workspace_bytes, void* stream) {
  if (out_peers == nullptr || flag_peers == nullptr || world < 1 || world > kMaxGatherWorld || rank < 0 || rank >= world)
    return fail(ERR_ARG, "qbits_mm_gather: need 1..8 peer buffers / flag arrays and 0 <= rank < world");
  QbitsArgs q{};
  q.a = a; q.packed = packed; q.scale = scale; q.shift = shift; q.bias = bias;
  q.m = m; q.n = n_local; q.k = k; q.ld = n_local * world; q.col0 = n_local * rank;
  q.group = group; q.bits = 4; q.dtype = dtype; q.shift_is_int = shift_is_int;
  q.workspace = workspace; q.workspace_bytes = workspace_bytes;
  // this rank's own buffer first (stores to local memory are issued before the NVLink ones)
  int cnt = 0;
  q.g.out_peer[cnt] = out_peers[rank];
  q.g.flag_peer[cnt++] = static_cast<uint32_t*>(flag_peers[rank]);
  for (int r = 0; r < world; ++r)
    if (r != rank) {
      q.g.out_peer[cnt] = out_peers[r];
      q.g.flag_peer[cnt++] = static_cast<uint32_t*>(flag_peers[r]);
    }
  for (int i = 0; i < cnt; ++i)
    if (q.g.out_peer[i] == nullptr || q.g.flag_peer[i] == nullptr) return fail(ERR_ARG, "qbits_mm_gather: null peer buffer");
  q.g.flags = q.g.flag_peer[0];
  q.g.n_out = cnt;
  q.g.world = world;
  q.g.rank = rank;
  q.g.wait_start = (wait_flags & QB200_GATHER_WAIT_INPUT) ? 1 : 0;
  q.g.wait_end = (wait_flags & QB200_GATHER_WAIT_OUTPUT) ? 1 : 0;
  q.out = q.g.out_peer[0];
  q.stream = static_cast<cudaStream_t>(stream);
  if (world == 1) {  // degenerate: an ordinary call into the caller's buffer
    q.g.n_out = 1;
  }
  return qbits_mm_impl(q);
}

}  // extern "C"
