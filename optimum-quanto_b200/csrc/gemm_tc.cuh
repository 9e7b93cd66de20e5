// Persistent, warp-specialised wgmma GEMM for the quantized-linear forward (Hopper, sm_90a).
//
//   out[m, n] = epilogue( sum_k A[m, k] * Wt[n, k] )
//
// One CTA per SM loops over BM x BN output tiles (BM = 64 per consumer warpgroup, BN = 128 or 256).  Roles:
//   warps [0, 4*MWG)  consumers      : one warpgroup per 64 rows of the tile issues wgmma (accumulators in registers)
//                                      and runs the epilogue (scale / bias / round / optional output quantisation)
//   warp 4*MWG        TMA producer   : A tiles (and W tiles when W is 8-bit and fed straight to the tensor core)
//   further warps     weight staging : (int4 / weight-only 8-bit) vector-load the packed weight bytes, unpack,
//                                      apply the per-group scale/shift with the reference's exact rounding order and
//                                      write the bf16/fp16 tile into shared memory in the 128B-swizzled K-major
//                                      layout the tensor core reads -- no separate dequantise launch, the
//                                      dequantised weight never exists in HBM.
//
// Shared-memory operand layout (both operands, K-major): a tile is `rows x 128 bytes`; row r lives at
// (r/8)*1024 + (r%8)*128 and its 16-byte chunk c is stored at chunk position c ^ (r%8)  (SWIZZLE_128B, the
// layout TMA produces and the wgmma descriptor in common.cuh describes).
#pragma once

#include <type_traits>

#include "common.cuh"
#include "gather.cuh"
#include "host_common.cuh"
#include "quantize_math.cuh"
#include "wgmma_pipe.cuh"

namespace qb {

// BYTES: int8 / fp8 weights converted in-kernel to the activation dtype; F8: fp8 activations AND weights converted
// in-kernel to bf16 (exact: every e4m3 / e5m2 value is a bf16 value), so that the products are exact and summed in fp32
enum class BSrc { TMA, INT4, BYTES, F8 };

struct GemmParams {
  // epilogue
  const void* scales;  // [N] in the output dtype, applied in fp32 to the accumulator (8-bit paths) or nullptr
  const void* bias;    // [N] in the output dtype or nullptr; added after the result is rounded (reference order)
  void* out;           // [M, ld] output of this rank (== g.out_peer[0])
  // Fused all-gather of a column-parallel linear (SURVEY 8e, gather.cuh): the epilogue stores every output tile into
  // g.n_out buffers -- this rank's and its peers' [M, ld] outputs, peer-mapped over NVLink -- at column offset `col0`,
  // and the kernel carries the rank synchronisation itself.  An ordinary call has g.n_out = 1, ld = N, col0 = 0.
  GatherInfo g;
  int ld;              // row pitch of the output buffers in elements
  int col0;            // first output column of this rank's slab
  int out_dt;          // DT_F32 / DT_F16 / DT_BF16
  int M, N, K;         // K in elements
  int num_m_blocks, num_n_blocks;
  // int4 weight source (BSrc::INT4): canonical quanto storage viewed as [N/2, K] bytes,
  // low nibble = out-feature n, high nibble = out-feature n + N/2 (tensor/packed.py:45-69)
  const uint8_t* wq;
  const void* wscale;  // [N * K / group]
  const void* wshift;  // same shape; weight dtype, or uint8 zero-point when shift_is_int
  int group;
  int group_log2;      // log2(group) when group is a power of two, else -1
  int shift_is_int;
  // 8-bit weight source (BSrc::BYTES): wq = W [N, K] int8 / e4m3 / e5m2, wscale = per-out-feature scales [N] in the
  // activation dtype; the staging warps write rnd(scale * W) exactly as the reference's python path does
  // (library/qbytes_mm.py:25-33), so the GEMM operands are bit-identical to the reference's
  int w_dt;
  const void* a;       // F8 only: the [M, K] fp8 activations, read by the staging warps
  // Fused output quantisation (SURVEY 8f rank 2: QModuleMixin.quantize_output, nn/qmodule.py:300-302, fused into the
  // epilogue): q_dt = DT_I8 / DT_E4M3 / DT_E5M2 (0 = off), q_scale = DEVICE pointer to the per-tensor output scale in
  // `out_dt`.  The result rounded to out_dt (+ bias, rounded) is divided by the scale in out_dt, rounded, clamped and
  // cast exactly like quanto::quantize_symmetric; `out` is then a [M, ld] buffer of BYTES.
  int q_dt;
  const void* q_scale;
  // BSrc::INT4: 1 = the epilogue stores each tile with TMA through `tmap_out` (one dense [M, N] output: g.n_out = 1,
  // ld = N, col0 = 0, N % 16 == 0); 0 = ordinary stores
  int epi_tma;
  int dbg;  // developer knock-outs (debug_flags(); always 0 in the release library, see QB_KO)
  // Batched int8 x int8 (GemmCfg::BATCH, quanto::qbytes_bmm): out[b] = A[b] @ B[b]^T, with rank-3 tensor maps
  // [batch, rows, K] for both operands.  num_n_blocks = batch * n_blocks_per_batch (tile t: m-block t % num_m_blocks,
  // then n-block, then batch); `out` is the dense [batch, M, N] output.  The output scale is the ONE scalar
  // rnd_out(scales[0] * scale_b[0]) (the two per-tensor activation scales).  a_batch_mul / b_batch_mul are 0 for an
  // operand broadcast over the batch (its tensor map has one batch), else 1.
  const void* scale_b;
  int n_blocks_per_batch;
  int a_batch_mul, b_batch_mul;
};

// ------------------------------------------------------------------------------------------------
// int4 -> bf16/fp16 with the reference's rounding order (tensor/qbits.py:34-45)
//   float shift: d = rnd(rnd(s*q) - z)            int shift: d = rnd(s * (q - zp))
// q enters as the magic-number pattern (bf16: 0x4300|q = 128+q, fp16: 0x6400|q = 1024+q), two per register.
// ------------------------------------------------------------------------------------------------
template <typename T>
struct Dq;

template <>
struct Dq<__nv_bfloat16> {
  using V2 = __nv_bfloat162;
  static constexpr uint32_t MAGIC_BYTES = 0x43434343u;
  struct Coef { V2 s, c, z; };  // float shift: c = -128*s ; int shift: c = 128 + zp
  // `zraw`: the shift's 16-bit payload (bf16 bits) or, for integer shifts, the zero-point byte
  __device__ __forceinline__ static Coef make_raw(__nv_bfloat16 s, uint16_t zraw, bool is_int) {
    Coef k;
    k.s = __bfloat162bfloat162(s);
    if (is_int) {
      const int zp = static_cast<int8_t>(static_cast<uint8_t>(zraw));
      k.c = __bfloat162bfloat162(__float2bfloat16_rn(128.f + static_cast<float>(zp)));
      k.z = k.c;
    } else {
      k.c = __hmul2_rn(k.s, __bfloat162bfloat162(__float2bfloat16_rn(-128.f)));
      k.z = __bfloat162bfloat162(__ushort_as_bfloat16(zraw));
    }
    return k;
  }
  __device__ static Coef make(__nv_bfloat16 s, const void* shift_ptr, int64_t idx, bool is_int) {
    const uint16_t zraw = is_int ? static_cast<uint16_t>(static_cast<const uint8_t*>(shift_ptr)[idx])
                                 : static_cast<const uint16_t*>(shift_ptr)[idx];
    return make_raw(s, zraw, is_int);
  }
  __device__ __forceinline__ static uint32_t cvt(uint32_t m, const Coef& k, bool is_int) {
    V2 v = *reinterpret_cast<V2*>(&m);
    V2 d;
    // the *_rn intrinsics forbid ptxas from contracting mul+sub into one fma (which would drop a rounding step)
    if (is_int) d = __hmul2_rn(k.s, __hsub2_rn(v, k.c));      // (128+q)-(128+zp) exact, one rounding
    else d = __hsub2_rn(__hfma2(k.s, v, k.c), k.z);           // s*(128+q) - 128*s == s*q exactly -> rnd ; then - z -> rnd
    return *reinterpret_cast<uint32_t*>(&d);
  }
};

template <>
struct Dq<__half> {
  using V2 = __half2;
  static constexpr uint32_t MAGIC_BYTES = 0x64646464u;
  struct Coef { V2 s, c, z; };  // c = 1024 (float shift) or 1024 + zp (int shift)
  __device__ __forceinline__ static Coef make_raw(__half s, uint16_t zraw, bool is_int) {
    Coef k;
    k.s = __half2half2(s);
    if (is_int) {
      const int zp = static_cast<int8_t>(static_cast<uint8_t>(zraw));
      k.c = __half2half2(__float2half_rn(1024.f + static_cast<float>(zp)));
      k.z = k.c;
    } else {
      k.c = __half2half2(__float2half_rn(1024.f));
      k.z = __half2half2(__ushort_as_half(zraw));
    }
    return k;
  }
  __device__ static Coef make(__half s, const void* shift_ptr, int64_t idx, bool is_int) {
    const uint16_t zraw = is_int ? static_cast<uint16_t>(static_cast<const uint8_t*>(shift_ptr)[idx])
                                 : static_cast<const uint16_t*>(shift_ptr)[idx];
    return make_raw(s, zraw, is_int);
  }
  __device__ __forceinline__ static uint32_t cvt(uint32_t m, const Coef& k, bool is_int) {
    V2 v = *reinterpret_cast<V2*>(&m);
    V2 d;
    if (is_int) d = __hmul2_rn(k.s, __hsub2_rn(v, k.c));
    else d = __hsub2_rn(__hmul2_rn(k.s, __hsub2_rn(v, k.c)), k.z);  // (1024+q)-1024 exact ; s*q -> rnd ; - z -> rnd
    return *reinterpret_cast<uint32_t*>(&d);
  }
};

// 16 packed bytes (16 k of two out-features) -> 2 x 8 registers of bf16x2 / half2 (natural k order).
// 7 integer ops + 8 (bf16) half-precision ops per 8 weights.
template <typename WT, bool ZP>
__device__ __forceinline__ void dequant16(const uint4& raw, const typename Dq<WT>::Coef& klo,
                                          const typename Dq<WT>::Coef& khi, uint32_t (&lo)[8], uint32_t (&hi)[8]) {
  using D = Dq<WT>;
  const uint32_t w4[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const uint32_t wl = w4[i] & 0x0F0F0F0Fu;
    const uint32_t wh = (w4[i] >> 4) & 0x0F0F0F0Fu;
    lo[2 * i + 0] = D::cvt(__byte_perm(wl, D::MAGIC_BYTES, 0x4140), klo, ZP);
    lo[2 * i + 1] = D::cvt(__byte_perm(wl, D::MAGIC_BYTES, 0x4342), klo, ZP);
    hi[2 * i + 0] = D::cvt(__byte_perm(wh, D::MAGIC_BYTES, 0x4140), khi, ZP);
    hi[2 * i + 1] = D::cvt(__byte_perm(wh, D::MAGIC_BYTES, 0x4342), khi, ZP);
  }
}

// The scale and shift of one group of a packed row's two out-features (low nibble: element ilo of the coefficient
// arrays, high nibble: ihi), as 16-bit payloads: the shift is in the weight dtype, or a uint8 zero-point when ZP.
struct CoefPair { uint16_t s_lo, s_hi, z_lo, z_hi; };
template <bool ZP>
__device__ __forceinline__ CoefPair load_coef_pair(const void* wscale, const void* wshift, size_t ilo, size_t ihi) {
  CoefPair c;
  c.s_lo = __ldg(static_cast<const uint16_t*>(wscale) + ilo);
  c.s_hi = __ldg(static_cast<const uint16_t*>(wscale) + ihi);
  if (ZP) {
    c.z_lo = __ldg(static_cast<const uint8_t*>(wshift) + ilo);
    c.z_hi = __ldg(static_cast<const uint8_t*>(wshift) + ihi);
  } else {
    c.z_lo = __ldg(static_cast<const uint16_t*>(wshift) + ilo);
    c.z_hi = __ldg(static_cast<const uint16_t*>(wshift) + ihi);
  }
  return c;
}

template <typename WT>
__device__ __forceinline__ WT bits_as(uint16_t b) {
  return *reinterpret_cast<const WT*>(&b);
}

// 64 packed bytes of one packed row (64 k of out-features n and n + N/2) -> two 128-byte operand rows in shared
// memory (SWIZZLE_128B: chunk c of a row lands at c ^ sw).  `klo/khi[1]` are used for k >= 32 when the group size
// is 32 (two groups inside the 64 k); otherwise index 0 serves all.
template <typename WT, bool ZP>
__device__ __forceinline__ void stage_rowpair_64k(const uint4 (&raw)[4], const typename Dq<WT>::Coef (&klo)[2],
                                                  const typename Dq<WT>::Coef (&khi)[2], uint32_t dst_lo,
                                                  uint32_t dst_hi, uint32_t sw) {
#pragma unroll
  for (int v = 0; v < 4; ++v) {
    constexpr int kHalf = 2;
    const int set = (v >= kHalf) ? 1 : 0;  // compile-time after unrolling (callers alias set 1 to set 0 if unused)
    uint32_t lo[8], hi[8];
    dequant16<WT, ZP>(raw[v], klo[set], khi[set], lo, hi);
    const uint32_t c0 = ((2u * v + 0u) ^ sw) << 4, c1 = ((2u * v + 1u) ^ sw) << 4;
    st_shared_v4(dst_lo + c0, lo[0], lo[1], lo[2], lo[3]);
    st_shared_v4(dst_lo + c1, lo[4], lo[5], lo[6], lo[7]);
    st_shared_v4(dst_hi + c0, hi[0], hi[1], hi[2], hi[3]);
    st_shared_v4(dst_hi + c1, hi[4], hi[5], hi[6], hi[7]);
  }
}

__device__ __forceinline__ void zero_rowpair_64k(uint32_t dst_lo, uint32_t dst_hi) {
#pragma unroll
  for (int c = 0; c < 8; ++c) {
    st_shared_v4(dst_lo + (c << 4), 0u, 0u, 0u, 0u);
    st_shared_v4(dst_hi + (c << 4), 0u, 0u, 0u, 0u);
  }
}

// 8-bit weights -> activation dtype, exactly (every int8 / e4m3 / e5m2 value is representable in bf16 and fp16),
// then one rounding multiply by the per-row scale: Ws = rnd(scale * W), the reference's operand.
template <typename WT>
__device__ __forceinline__ uint32_t pack2(float a, float b);
template <>
__device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
template <>
__device__ __forceinline__ uint32_t pack2<__half>(float a, float b) {
  __half2 t = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}
template <typename WT>
__device__ __forceinline__ uint32_t mul2_rn(uint32_t v, uint32_t s2);
template <>
__device__ __forceinline__ uint32_t mul2_rn<__nv_bfloat16>(uint32_t v, uint32_t s2) {
  __nv_bfloat162 r = __hmul2_rn(*reinterpret_cast<__nv_bfloat162*>(&s2), *reinterpret_cast<__nv_bfloat162*>(&v));
  return *reinterpret_cast<uint32_t*>(&r);
}
template <>
__device__ __forceinline__ uint32_t mul2_rn<__half>(uint32_t v, uint32_t s2) {
  __half2 r = __hmul2_rn(*reinterpret_cast<__half2*>(&s2), *reinterpret_cast<__half2*>(&v));
  return *reinterpret_cast<uint32_t*>(&r);
}

// 4 bytes (k .. k+3 of one weight row) -> 2 registers of WT pairs, scaled.
template <typename WT, int WKIND>
__device__ __forceinline__ void cvt_bytes4(uint32_t w, uint32_t s2, uint32_t& o01, uint32_t& o23) {
  if constexpr (WKIND == 0) {
    // int8: byte b -> float(2^23 + (b ^ 0x80)) - (2^23 + 128) == b exactly
    const uint32_t u = w ^ 0x80808080u;
    const float f0 = __uint_as_float(__byte_perm(u, 0x4B000000u, 0x7440)) - 8388736.f;
    const float f1 = __uint_as_float(__byte_perm(u, 0x4B000000u, 0x7441)) - 8388736.f;
    const float f2 = __uint_as_float(__byte_perm(u, 0x4B000000u, 0x7442)) - 8388736.f;
    const float f3 = __uint_as_float(__byte_perm(u, 0x4B000000u, 0x7443)) - 8388736.f;
    o01 = mul2_rn<WT>(pack2<WT>(f0, f1), s2);
    o23 = mul2_rn<WT>(pack2<WT>(f2, f3), s2);
  } else if constexpr (WKIND == 3) {
    // float8_e4m3fnuz: bits << 7 in the fp16 fields = value / 128 (see e4m3fnuz_to_float); 0x80 = NaN
    const uint32_t t01 = __byte_perm(w, 0u, 0x4140), t23 = __byte_perm(w, 0u, 0x4342);  // one byte per 16-bit lane
    uint32_t h01 = ((t01 & 0x007F007Fu) << 7) | ((t01 & 0x00800080u) << 8);
    uint32_t h23 = ((t23 & 0x007F007Fu) << 7) | ((t23 & 0x00800080u) << 8);
    h01 |= __vcmpeq2(t01, 0x00800080u) & 0x7FFF7FFFu;
    h23 |= __vcmpeq2(t23, 0x00800080u) & 0x7FFF7FFFu;
    const __half2 k128 = __float2half2_rn(128.f);
    const __half2 a2 = __hmul2(*reinterpret_cast<__half2*>(&h01), k128), b2 = __hmul2(*reinterpret_cast<__half2*>(&h23), k128);
    if constexpr (std::is_same<WT, __half>::value) {
      o01 = mul2_rn<WT>(*reinterpret_cast<const uint32_t*>(&a2), s2);
      o23 = mul2_rn<WT>(*reinterpret_cast<const uint32_t*>(&b2), s2);
    } else {
      const float2 a = __half22float2(a2), b = __half22float2(b2);
      o01 = mul2_rn<WT>(pack2<WT>(a.x, a.y), s2);
      o23 = mul2_rn<WT>(pack2<WT>(b.x, b.y), s2);
    }
  } else {
    constexpr __nv_fp8_interpretation_t KIND = (WKIND == 1) ? __NV_E4M3 : __NV_E5M2;
    const __half2_raw h01 = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w & 0xFFFFu), KIND);
    const __half2_raw h23 = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w >> 16), KIND);
    if constexpr (std::is_same<WT, __half>::value) {
      uint32_t a = static_cast<uint32_t>(h01.x) | (static_cast<uint32_t>(h01.y) << 16);
      uint32_t b = static_cast<uint32_t>(h23.x) | (static_cast<uint32_t>(h23.y) << 16);
      o01 = mul2_rn<WT>(a, s2);
      o23 = mul2_rn<WT>(b, s2);
    } else {
      const float2 a = __half22float2(__half2(h01));
      const float2 b = __half22float2(__half2(h23));
      o01 = mul2_rn<WT>(pack2<WT>(a.x, a.y), s2);
      o23 = mul2_rn<WT>(pack2<WT>(b.x, b.y), s2);
    }
  }
}

// 64 bytes of one weight row -> one 128-byte operand row (SWIZZLE_128B)
template <typename WT, int WKIND>
__device__ __forceinline__ void stage_row_64k(const uint4 (&raw)[4], uint32_t s2, uint32_t dst, uint32_t sw) {
#pragma unroll
  for (int v = 0; v < 4; ++v) {
    uint32_t o[8];
    cvt_bytes4<WT, WKIND>(raw[v].x, s2, o[0], o[1]);
    cvt_bytes4<WT, WKIND>(raw[v].y, s2, o[2], o[3]);
    cvt_bytes4<WT, WKIND>(raw[v].z, s2, o[4], o[5]);
    cvt_bytes4<WT, WKIND>(raw[v].w, s2, o[6], o[7]);
    st_shared_v4(dst + (((2u * v + 0u) ^ sw) << 4), o[0], o[1], o[2], o[3]);
    st_shared_v4(dst + (((2u * v + 1u) ^ sw) << 4), o[4], o[5], o[6], o[7]);
  }
}

// ------------------------------------------------------------------------------------------------
// Kernel configuration
// ------------------------------------------------------------------------------------------------
// KIND_: MMA operand kind (F16 / BF16, or I8 for int8 x int8).  MWG_: consumer warpgroups (BM = 64 * MWG_).
// WT_: staged element type (INT4 / BYTES / F8).
// BATCH_: the batched int8 x int8 product of quanto::qbytes_bmm (see GemmParams).
template <MmaKind KIND_, BSrc BSRC_, int MWG_, int BN_, typename WT_ = __nv_bfloat16, bool ZP_ = false, int WKIND_ = 0,
          int AKIND_ = 0, bool BATCH_ = false>
struct GemmCfg {
  static constexpr MmaKind KIND = KIND_;
  static constexpr BSrc BSRC = BSRC_;
  static constexpr bool BATCH = BATCH_;
  static constexpr bool ZP = ZP_;       // INT4 only: shift is an integer zero-point (compile-time: keeps the hot loop lean)
  static constexpr int WKIND = WKIND_;  // BYTES / F8: weight bytes: 0 int8, 1 float8_e4m3fn, 2 float8_e5m2, 3 float8_e4m3fnuz
  static constexpr int AKIND = AKIND_;  // F8: activation bytes, same codes
  using WT = WT_;
  static constexpr int MWG = MWG_;
  static constexpr int BM = 64 * MWG;
  static constexpr int BN = BN_;
  static constexpr bool IS_INT = (KIND == MmaKind::I8);
  static constexpr int NACC = BN / 2;   // accumulator registers per consumer thread
  static constexpr int KBYTES = 128;    // K extent of one pipeline stage in bytes = one swizzle atom
  static constexpr int A_TILE = BM * KBYTES;
  static constexpr int B_TILE = BN * KBYTES;
  // staged weights: one staging group (BN/64 warps: one thread per packed int4 row, or per two 8-bit rows -- and for F8
  // per one or two activation rows) per stage slot.  3 slots keep the CTA at 15 warps, which leaves 128 registers per thread (the consumers hold 64 accumulators).
  static constexpr int NSTAGES =
      (BSRC == BSrc::TMA) ? ((192 * 1024) / (A_TILE + B_TILE) > 8 ? 8 : (192 * 1024) / (A_TILE + B_TILE)) : 3;
  // int4: one 64 x BN output staging tile of the activation dtype per consumer warpgroup (int4_epilogue)
  static constexpr int EPI_TILE = (BSRC == BSrc::INT4) ? 64 * BN * 2 : 0;
  // the TMA producer's arrive (A tile, and W for TMA) + one per staging warp; F8 stages both operands without TMA
  using Pipe = PipeLayout<MWG, NSTAGES, A_TILE, B_TILE, (BSRC == BSrc::TMA) ? 0 : BN / 64, (BSRC == BSrc::F8) ? 0 : 1,
                          MWG * EPI_TILE>;
  static_assert(BN == 128 || (BN == 256 && IS_INT && BSRC == BSrc::TMA), "wgmma tile width");
  static_assert(BSRC == BSrc::TMA || KIND == MmaKind::F16 || KIND == MmaKind::BF16, "staged weights are 16-bit");
  static_assert(!BATCH || (IS_INT && BSRC == BSrc::TMA), "batched: int8 x int8 with both operands fed by TMA");
};

// ------------------------------------------------------------------------------------------------
// Epilogue, one pair of adjacent accumulator columns of one output row (the wgmma fragment holds pairs):
//   8-bit operands : rnd_OT(acc * scale[n]) (+ bias, rounded) -- the reference's qbytes_mm + bias order;
//                    with q_dt != 0 that result is then quantised like quanto::quantize_symmetric and stored as bytes
//   16-bit operands: rnd_OT(acc) (+ bias, rounded)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float load_out_dt_as_float(const void* base, int dt, int i) {
  if (dt == DT_BF16) return __bfloat162float(static_cast<const __nv_bfloat16*>(base)[i]);
  if (dt == DT_F16) return __half2float(static_cast<const __half*>(base)[i]);
  return static_cast<const float*>(base)[i];
}

template <typename OT>
__device__ __forceinline__ void store_pair(OT* dst, float a, float b, bool two, bool vec) {
  if (two && vec) {
    if constexpr (sizeof(OT) == 2) *reinterpret_cast<uint32_t*>(dst) = pack2<OT>(a, b);
    else *reinterpret_cast<float2*>(dst) = make_float2(a, b);
  } else {
    dst[0] = from_float<OT>(a);
    if (two) dst[1] = from_float<OT>(b);
  }
}

// f0, f1: accumulator values of output features n, n + 1 (n + 1 only when `two`); row_off = row * ld + col0.
// PER_N = false: the caller has applied the scale already (the batched kernel's one scalar), p.scales is not read.
template <typename OT, bool ALLOW_Q, bool PER_N = true>
__device__ __forceinline__ void epilogue_pair_t(const GemmParams& p, size_t row_off, int n, bool two, float f0, float f1) {
  if (PER_N && p.scales != nullptr) {
    f0 = __fmul_rn(f0, load_out_dt_as_float(p.scales, p.out_dt, n));
    if (two) f1 = __fmul_rn(f1, load_out_dt_as_float(p.scales, p.out_dt, n + 1));
  }
  rnd_pair<OT>(f0, f1);
  if (p.bias != nullptr) {
    f0 = __fadd_rn(f0, load_out_dt_as_float(p.bias, p.out_dt, n));
    if (two) f1 = __fadd_rn(f1, load_out_dt_as_float(p.bias, p.out_dt, n + 1));
    rnd_pair<OT>(f0, f1);
  }
  if constexpr (ALLOW_Q) {
    if (p.q_dt != 0) {
      const float qs = to_float<OT>(*static_cast<const OT*>(p.q_scale));
      if (rcp_is_safe<OT>(qs)) {
        const float qr = __frcp_rn(qs);
        f0 = __fmul_rn(f0, qr);
        f1 = __fmul_rn(f1, qr);
      } else {
        f0 = __fdiv_rn(f0, qs);
        f1 = __fdiv_rn(f1, qs);
      }
      rnd_pair<OT>(f0, f1);
      uint8_t q0, q1;
      if (p.q_dt == DT_I8) { q0 = quantize_one<DT_I8>(f0); q1 = quantize_one<DT_I8>(f1); }
      else if (p.q_dt == DT_E4M3) { q0 = quantize_one<DT_E4M3>(f0); q1 = quantize_one<DT_E4M3>(f1); }
      else { q0 = quantize_one<DT_E5M2>(f0); q1 = quantize_one<DT_E5M2>(f1); }
      for (int q = 0; q < p.g.n_out; ++q) {
        uint8_t* dst = static_cast<uint8_t*>(p.g.out_peer[q]) + row_off + n;
        dst[0] = q0;
        if (two) dst[1] = q1;
      }
      return;
    }
  }
  const bool vec = ((row_off + n) * sizeof(OT)) % (2 * sizeof(OT)) == 0;
  for (int q = 0; q < p.g.n_out; ++q) store_pair<OT>(static_cast<OT*>(p.g.out_peer[q]) + row_off + n, f0, f1, two, vec);
}

template <bool ALLOW_Q, bool PER_N = true>
__device__ __forceinline__ void epilogue_pair(const GemmParams& p, size_t row_off, int n, bool two, float f0, float f1) {
  if (p.out_dt == DT_BF16) epilogue_pair_t<__nv_bfloat16, ALLOW_Q, PER_N>(p, row_off, n, two, f0, f1);
  else if (p.out_dt == DT_F16) epilogue_pair_t<__half, ALLOW_Q, PER_N>(p, row_off, n, two, f0, f1);
  else epilogue_pair_t<float, ALLOW_Q, PER_N>(p, row_off, n, two, f0, f1);
}

// rnd_dt(sa * sb) of two one-element scales of dtype `dt`: the output scale of the reference's int8 bmm
// (tensor/activations/qbytes_ops.py:185, `input._scale * other._scale` in the scale dtype, then widened to fp32).
__device__ __forceinline__ float scalar_scale_product(const void* sa, const void* sb, int dt) {
  const float s = __fmul_rn(load_out_dt_as_float(sa, dt, 0), load_out_dt_as_float(sb, dt, 0));
  if (dt == DT_BF16) return rnd<__nv_bfloat16>(s);
  if (dt == DT_F16) return rnd<__half>(s);
  return s;
}

// Epilogue of the int4 kernels (output dtype OT = the 16-bit activation dtype), one consumer warpgroup's 64-row slice
// of a 64 x 128 tile.  The tile's columns [0, 64) are the low-nibble out-features n_blk * 64 + c, its columns
// [64, 128) the high-nibble ones N/2 + n_blk * 64 + c - 64.
//   1. The warpgroup rounds its accumulators, rnd_OT(acc) (+ bias, rounded), into its staging tile `stile`: two planes
//      of 64 rows x 64 columns (low- and high-nibble columns), each row 128 bytes with the 128-byte swizzle.
//   2. p.epi_tma: one thread stores the two planes with TMA into the output seen as [M, 2, N/2] (`tmap_out`, box 64
//      columns x 1 plane x 64 rows); TMA drops what lies past M or past the end of a plane.  The store completes while
//      the next tile's mainloop runs; the next epilogue waits until it has read the staging tile.
//      Otherwise the warpgroup copies the tile out with ordinary, bounds-checked stores into every output buffer of
//      the fused gather, at the row pitch `ld` and column offset `col0`.
constexpr int kInt4EpiPlane = 64 * 128;  // bytes of one staging plane
template <typename OT>
__device__ __forceinline__ void int4_epilogue(const GemmParams& p, const CUtensorMap* tmap_out, const float (&acc)[64],
                                              uint32_t stile, int row0, int n_blk, int wg) {
  const int t = threadIdx.x & 127;
  const int lane = t & 31;
  const int half_n = p.N / 2;
  const OT* bias = static_cast<const OT*>(p.bias);
  // the staging tile is free: the previous tile's TMA store has read it, and every thread has finished copying it out
  if (t == 0) bulk_wait_group_read<0>();
  named_bar_sync(1 + wg, 128);
  // fragment (common.cuh): acc[4 j + 2 h + e] is row 16 (t / 32) + lane / 4 + 8 h, column 8 j + 2 (lane % 4) + e.  Row r
  // of a plane lives at r * 128 with 16-byte chunk c at c ^ (r % 8), and r % 8 == lane / 4: the 32 lanes of a warp
  // write 32 different banks.
  const uint32_t sw = static_cast<uint32_t>(lane) >> 2;
  const uint32_t row_addr = stile + static_cast<uint32_t>((t >> 5) * 16 + (lane >> 2)) * 128 + (lane & 3) * 4;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int n = (j < 8 ? 0 : half_n) + n_blk * 64 + 8 * (j & 7) + 2 * (lane & 3);
    const int n_limit = j < 8 ? half_n : p.N;
    float b0 = 0.f, b1 = 0.f;
    if (bias != nullptr) {
      if (n < n_limit) b0 = to_float<OT>(bias[n]);
      if (n + 1 < n_limit) b1 = to_float<OT>(bias[n + 1]);
    }
    const uint32_t a = row_addr + (j >> 3) * kInt4EpiPlane + ((static_cast<uint32_t>(j & 7) ^ sw) << 4);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
      rnd_pair<OT>(f0, f1);
      if (bias != nullptr) {
        f0 = __fadd_rn(f0, b0);
        f1 = __fadd_rn(f1, b1);
        rnd_pair<OT>(f0, f1);
      }
      st_shared_u32(a + h * 8 * 128, pack2<OT>(f0, f1));
    }
  }
  fence_proxy_async_smem();  // the tile's generic-proxy writes -> visible to the TMA store
  named_bar_sync(1 + wg, 128);
  if (p.epi_tma) {
    if (t == 0 && row0 < p.M) {
      tma_store_3d(tmap_out, stile, n_blk * 64, 0, row0);
      tma_store_3d(tmap_out, stile + kInt4EpiPlane, n_blk * 64, 1, row0);
      bulk_commit_group();
    }
    return;
  }
  // copy-out: thread t moves column pair 2 (t % 64) of rows t / 64, t / 64 + 2, ...: a warp reads one 128-byte plane row
  // and writes 32 consecutive pairs
  const int c = 2 * (t & 63);
  const int plane = c >> 6, pc = c & 63;
  const int n = (plane ? half_n : 0) + n_blk * 64 + pc;
  const int n_limit = plane ? p.N : half_n;
  if (n >= n_limit) return;
  const bool two = n + 1 < n_limit;
  const uint32_t src = stile + plane * kInt4EpiPlane + (pc & 7) * 2;
  for (int r = t >> 6; r < 64 && row0 + r < p.M; r += 2) {
    const uint32_t v = ld_shared_u32(src + r * 128 + ((static_cast<uint32_t>(pc >> 3) ^ (r & 7)) << 4));
    const size_t off = static_cast<size_t>(row0 + r) * p.ld + p.col0 + n;
    const bool vec = (off * sizeof(OT)) % (2 * sizeof(OT)) == 0;
    for (int q = 0; q < p.g.n_out; ++q) {
      uint16_t* dst = static_cast<uint16_t*>(p.g.out_peer[q]) + off;
      if (two && vec) {
        *reinterpret_cast<uint32_t*>(dst) = v;
      } else {
        dst[0] = static_cast<uint16_t>(v);
        if (two) dst[1] = static_cast<uint16_t>(v >> 16);
      }
    }
  }
}

// The weight-staging warps of gemm_tc_kernel and conv_tc_kernel (conv_tc.cuh): int4 or 8-bit weights -> the stage's
// 16-bit B tile, one staging group per stage slot (wgmma_pipe.cuh: StagingThread).
template <class Cfg>
__device__ __forceinline__ void stage_weights(const WgmmaPipe<typename Cfg::Pipe>& pipe, const GemmParams& p,
                                              int num_tiles, int kblocks) {
  using L = typename Cfg::Pipe;
  constexpr int BN = Cfg::BN;
  if constexpr (Cfg::BSRC == BSrc::INT4) {
    // ------------------------------------------------------------------ weight staging: int4 -> WT tile
    StagingThread<L> sg(pipe, num_tiles, kblocks);
    const int r = sg.r;
    const uint32_t sw = static_cast<uint32_t>(r) & 7;
    using WT = typename Cfg::WT;
    using D = Dq<WT>;
    constexpr bool ZP = Cfg::ZP;
    constexpr int ROWP = BN / 2;  // packed rows per tile, one per thread of the group
    static_assert(ROWP == StagingThread<L>::GT, "one staging thread per packed row");
    const int half_n = p.N / 2;
    const int groups_per_row = p.K / p.group;
    // A group that is not a multiple of 64 (32, 96, 160, ...) can change at the middle of a 64-k stage: two (scale,
    // shift) pairs per stage, one per 32-k half (a half lies inside one group: the group is a multiple of 32)
    const bool two_sets = p.group % 64 != 0;

    struct Pre {
      uint4 raw[4];
      WT s_lo[2], s_hi[2];
      uint16_t z_lo[2], z_hi[2];
      bool ok;
    };
    auto load_pre = [&](Pre& pr, const StageSeq<L::NSTAGES>& seq) {
      const int rp = (seq.tile / p.num_m_blocks) * ROWP + r;
      const int kbase = seq.kb * 64;
      pr.ok = rp < half_n && kbase < p.K;
      if (pr.ok) {
        const uint8_t* src = p.wq + static_cast<size_t>(rp) * p.K + kbase;
#pragma unroll
        for (int v = 0; v < 4; ++v)
          pr.raw[v] = (kbase + v * 16 < p.K) ? __ldg(reinterpret_cast<const uint4*>(src + v * 16)) : make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int s = 0; s < 2; ++s) {
          if (s == 1 && !two_sets) break;
          if (s == 1 && kbase + 32 >= p.K) {
            // K tail (K % 64 == 32 with groups of 32): the second half of the stage lies beyond K -- its activations are
            // zero-filled, but its coefficients would be read past the row (past the ARRAY for the last row: NaN bits
            // there turn 0 * w into NaN)
            pr.s_lo[1] = pr.s_lo[0]; pr.s_hi[1] = pr.s_hi[0]; pr.z_lo[1] = pr.z_lo[0]; pr.z_hi[1] = pr.z_hi[0];
            break;
          }
          const int ks = kbase + 32 * s;  // first k of the half
          const int gs = (p.group_log2 >= 0) ? (ks >> p.group_log2) : (ks / p.group);
          const size_t ilo = static_cast<size_t>(rp) * groups_per_row + gs;
          const size_t ihi = ilo + static_cast<size_t>(half_n) * groups_per_row;
          const CoefPair c = load_coef_pair<ZP>(p.wscale, p.wshift, ilo, ihi);
          pr.s_lo[s] = bits_as<WT>(c.s_lo);
          pr.s_hi[s] = bits_as<WT>(c.s_hi);
          pr.z_lo[s] = c.z_lo;
          pr.z_hi[s] = c.z_hi;
        }
      }
    };

    const uint32_t off_lo = (static_cast<uint32_t>(r) >> 3) * 1024 + (static_cast<uint32_t>(r) & 7) * 128;
    const uint32_t off_hi = off_lo + (ROWP / 8) * 1024;
    sg.template run_ping_pong<Pre>(load_pre, [&](const Pre& cur) {
      sg.wait_empty();
      if (cur.ok) {
        typename D::Coef klo[2], khi[2];
        klo[0] = D::make_raw(cur.s_lo[0], cur.z_lo[0], ZP);
        khi[0] = D::make_raw(cur.s_hi[0], cur.z_hi[0], ZP);
        if (two_sets) {
          klo[1] = D::make_raw(cur.s_lo[1], cur.z_lo[1], ZP);
          khi[1] = D::make_raw(cur.s_hi[1], cur.z_hi[1], ZP);
        } else {
          klo[1] = klo[0];
          khi[1] = khi[0];
        }
        stage_rowpair_64k<WT, ZP>(cur.raw, klo, khi, sg.bt + off_lo, sg.bt + off_hi, sw);
      } else {
        zero_rowpair_64k(sg.bt + off_lo, sg.bt + off_hi);
      }
      sg.publish();
    });
  } else if constexpr (Cfg::BSRC == BSrc::BYTES || Cfg::BSRC == BSrc::F8) {
    // ------------------------------------------------------------------ weight staging: 8-bit weights (int8 / fp8) ->
    // activation dtype, scale pre-applied (reference rounding order); F8: the weights unscaled (the scale is applied to
    // the fp32 result) and the activation rows of the tile as well
    StagingThread<L> sg(pipe, num_tiles, kblocks);
    constexpr int GT = StagingThread<L>::GT;
    const int r = sg.r;
    const uint32_t sw = static_cast<uint32_t>(r) & 7;
    using WT = typename Cfg::WT;
    static_assert(GT == BN / 2, "thread r converts weight rows r and r + BN/2");
    const WT* scale = static_cast<const WT*>(p.wscale);
    struct PreB {
      uint4 raw0[4], raw1[4];
    };
    auto load_pre = [&](PreB& pr, const StageSeq<L::NSTAGES>& seq) {
      const int n0 = (seq.tile / p.num_m_blocks) * BN + r;
      const int n1 = n0 + GT;
      const int kbase = seq.kb * 64;
#pragma unroll
      for (int v = 0; v < 4; ++v) {
        const bool kok = kbase + v * 16 < p.K;
        pr.raw0[v] = (n0 < p.N && kok) ? __ldg(reinterpret_cast<const uint4*>(p.wq + static_cast<size_t>(n0) * p.K + kbase) + v)
                                       : make_uint4(0, 0, 0, 0);
        pr.raw1[v] = (n1 < p.N && kok) ? __ldg(reinterpret_cast<const uint4*>(p.wq + static_cast<size_t>(n1) * p.K + kbase) + v)
                                       : make_uint4(0, 0, 0, 0);
      }
    };
    const uint32_t off0 = (static_cast<uint32_t>(r) >> 3) * 1024 + (static_cast<uint32_t>(r) & 7) * 128;
    const uint32_t off1 = off0 + (GT / 8) * 1024;
    int c_tile = -1;
    uint32_t s2_0 = 0, s2_1 = 0;
    auto process = [&](const PreB& cur, const StageSeq<L::NSTAGES>& seq) {
      if (Cfg::BSRC == BSrc::F8) {
        s2_0 = s2_1 = 0x3F803F80u;  // bf16 1.0 pair: the conversion alone, exact
      } else if (seq.tile != c_tile) {  // new tile: (re)load the two per-row scales (zero rows beyond N contribute exact zeros)
        c_tile = seq.tile;
        const int n0 = (c_tile / p.num_m_blocks) * BN + r;
        const int n1 = n0 + GT;
        const WT z = from_float<WT>(0.f);
        const WT a = (n0 < p.N) ? scale[n0] : z, b = (n1 < p.N) ? scale[n1] : z;
        const uint16_t ab = *reinterpret_cast<const uint16_t*>(&a), bb = *reinterpret_cast<const uint16_t*>(&b);
        s2_0 = static_cast<uint32_t>(ab) * 0x00010001u;
        s2_1 = static_cast<uint32_t>(bb) * 0x00010001u;
      }
      sg.wait_empty();
      stage_row_64k<WT, Cfg::WKIND>(cur.raw0, s2_0, sg.bt + off0, sw);
      stage_row_64k<WT, Cfg::WKIND>(cur.raw1, s2_1, sg.bt + off1, sw);
      if constexpr (Cfg::BSRC == BSrc::F8) {
        // activation rows r and r + 64 of the tile (BM = 64 or 128), loaded here rather than prefetched: the staging
        // thread has no registers left for a second pair of ping-pong buffers
        const int kbase = seq.kb * 64;
        const uint32_t at = sg.bt - Cfg::A_TILE;
#pragma unroll
        for (int h = 0; h < Cfg::BM / 64; ++h) {
          const int ar = r + 64 * h;
          const int m = (seq.tile % p.num_m_blocks) * Cfg::BM + ar;
          uint4 raw[4];
#pragma unroll
          for (int v = 0; v < 4; ++v)
            raw[v] = (m < p.M && kbase + v * 16 < p.K)
                         ? __ldg(reinterpret_cast<const uint4*>(static_cast<const uint8_t*>(p.a) + static_cast<size_t>(m) * p.K + kbase) + v)
                         : make_uint4(0, 0, 0, 0);
          const uint32_t aoff = (static_cast<uint32_t>(ar) >> 3) * 1024 + (static_cast<uint32_t>(ar) & 7) * 128;
          stage_row_64k<WT, Cfg::AKIND>(raw, 0x3F803F80u, at + aoff, sw);
        }
      }
      sg.publish();
    };
    // F8: one stage in registers at a time, the activation rows of the stage need the registers of a second buffer
    if constexpr (Cfg::BSRC == BSrc::F8) sg.template run_single<PreB>(load_pre, process);
    else sg.template run_ping_pong<PreB>(load_pre, process);
  }
}

// ------------------------------------------------------------------------------------------------
// The kernel
// ------------------------------------------------------------------------------------------------
template <class Cfg>
__global__ void __launch_bounds__(Cfg::Pipe::NTHREADS, 1)
    gemm_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_b,
                   const __grid_constant__ CUtensorMap tmap_out, const GemmParams p) {
  using L = typename Cfg::Pipe;
  constexpr int BN = Cfg::BN;

  const auto pipe = WgmmaPipe<L>::init([&] {
    tma_prefetch_desc(&tmap_a);
    if constexpr (Cfg::BSRC == BSrc::TMA) tma_prefetch_desc(&tmap_b);
    if constexpr (Cfg::BSRC == BSrc::INT4)
      if (p.epi_tma) tma_prefetch_desc(&tmap_out);
  });

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int num_tiles = p.num_m_blocks * p.num_n_blocks;
  constexpr int A_ELEM = (Cfg::KIND == MmaKind::F16 || Cfg::KIND == MmaKind::BF16) ? 2 : 1;
  constexpr int KELEMS = Cfg::KBYTES / A_ELEM;  // K elements per stage
  const int kblocks = (p.K + KELEMS - 1) / KELEMS;

  if (warp < L::PRODUCER_WARP) {
    // ------------------------------------------------------------------ consumers: wgmma + epilogue
    const int wg = warp >> 2;
    using AccT = typename std::conditional<Cfg::IS_INT, uint32_t, float>::type;
    AccT acc[Cfg::NACC];
    RingPos<L::NSTAGES> pos;
    float s_ab = 0.f;
    if constexpr (Cfg::BATCH) s_ab = scalar_scale_product(p.scales, p.scale_b, p.out_dt);
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile % p.num_m_blocks;
      int n_blk = tile / p.num_m_blocks;
      size_t out_base = 0;  // first element of the tile's batch in the output
      if constexpr (Cfg::BATCH) {
        const int b = n_blk / p.n_blocks_per_batch;
        n_blk -= b * p.n_blocks_per_batch;
        out_base = static_cast<size_t>(b) * p.M * p.ld;
      }
      pipe.consume_tile(pos, kblocks, acc, [&](uint32_t aa, uint32_t bb, bool accumulate) {
        wgmma_slab<Cfg::KIND, BN>(acc, aa, bb, accumulate);
      });
      if constexpr (Cfg::BSRC == BSrc::INT4) {
        int4_epilogue<typename Cfg::WT>(p, &tmap_out, acc, pipe.epi + wg * Cfg::EPI_TILE, m_blk * Cfg::BM + wg * 64,
                                        n_blk, wg);
      } else {
        // epilogue straight from the fragment: thread holds rows r0 and r0 + 8, column pairs 8 j + 2 (lane % 4)
        const int r0 = m_blk * Cfg::BM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int row = r0 + 8 * h;
          if (row >= p.M) continue;
          const size_t row_off = out_base + static_cast<size_t>(row) * p.ld + p.col0;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int n = n_blk * BN + 8 * j + 2 * (lane & 3);
            if (n >= p.N) continue;
            float f0, f1;
            if constexpr (Cfg::IS_INT) {
              f0 = __int2float_rn(static_cast<int>(acc[4 * j + 2 * h]));
              f1 = __int2float_rn(static_cast<int>(acc[4 * j + 2 * h + 1]));
            } else {
              f0 = acc[4 * j + 2 * h];
              f1 = acc[4 * j + 2 * h + 1];
            }
            if constexpr (Cfg::BATCH) {
              f0 = __fmul_rn(f0, s_ab);
              f1 = __fmul_rn(f1, s_ab);
              epilogue_pair<false, false>(p, row_off, n, n + 1 < p.N, f0, f1);
            } else {
              epilogue_pair<Cfg::BSRC == BSrc::TMA || Cfg::BSRC == BSrc::F8>(p, row_off, n, n + 1 < p.N, f0, f1);
            }
          }
        }
      }
    }
    if constexpr (Cfg::BSRC == BSrc::INT4)
      if ((threadIdx.x & 127) == 0) bulk_wait_group_all();  // the last tile's TMA store has completed
    if (p.g.n_out > 1) __threadfence_system();  // this thread's peer stores are performed before the rank signals
  } else if (warp == L::PRODUCER_WARP) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0 && Cfg::BSRC != BSrc::F8) {
      constexpr uint32_t tx_bytes = Cfg::A_TILE + (Cfg::BSRC == BSrc::TMA ? Cfg::B_TILE : 0);
      gather_wait_start(p.g);  // the activation may be the gathered output of the previous linear
      pipe.produce(num_tiles, p.num_m_blocks, kblocks, tx_bytes, [&](uint8_t* dst, uint64_t* bar, int m_blk, int n_blk, int kb) {
        if constexpr (Cfg::BATCH) {
          const int b = n_blk / p.n_blocks_per_batch;
          tma_load_3d(dst, &tmap_a, bar, kb * KELEMS, m_blk * Cfg::BM, b * p.a_batch_mul);
          tma_load_3d(dst + Cfg::A_TILE, &tmap_b, bar, kb * KELEMS, (n_blk - b * p.n_blocks_per_batch) * BN,
                      b * p.b_batch_mul);
        } else {
          tma_load_2d(dst, &tmap_a, bar, kb * KELEMS, m_blk * Cfg::BM);
          if constexpr (Cfg::BSRC == BSrc::TMA) tma_load_2d(dst + Cfg::A_TILE, &tmap_b, bar, kb * KELEMS, n_blk * BN);
        }
      });
    }
  } else if constexpr (Cfg::BSRC != BSrc::TMA) {
    stage_weights<Cfg>(pipe, p, num_tiles, kblocks);
  }

  __syncthreads();
  if (threadIdx.x == 0) gather_signal_end(p.g);  // fused all-gather: publish "this rank's slab has landed everywhere"
}

// ------------------------------------------------------------------------------------------------
// The int4 forward, swap-AB with the dequantised weight as the REGISTER operand of wgmma:
//
//   out^T[n, m] = sum_k Wdeq[n, k] * x[m, k]
//
// A tile is PR packed rows (out-features n and n + N/2 of each) x T tokens: PR = 128 at T = 64 and 128, PR = 64 at
// T = 256 (the MACs of T = 128; one m64n256k16 per step takes the dequantised values two m64n128k16 took).
// Roles:
//   warps 0-7      consumers   : warpgroup wg owns NF 64-row wgmma fragments (NF = 1 at T = 256, else 2), fragment
//                                f = packed rows 32 (NF wg + f) + 8 w + g of warp w, lane 4 g + c.  Per k16 step a
//                                thread reads its packed row's 4 bytes from shared memory, dequantises them with the
//                                Dq arithmetic (low nibble -> fragment row g, high nibble -> row g + 8: each packed
//                                byte feeds two rows) and issues m64 x T x k16 with A from registers and the
//                                activations (B) from shared memory.  The next step is dequantised while the MMA runs.
//   warp 8, lane 0 TMA producer: the activation box [T][64 k] (128B swizzle) and the packed box [PR][64 bytes] (64B
//                                swizzle: 16-byte chunk s of row r at s ^ ((r >> 1) & 3), so the 8 rows a warp reads
//                                per instruction hit 8 different bank groups)
//   warp 9         coefficients: the stage's scales and shifts, as 4-byte cp.async of the aligned word holding each
//                                value, completing on the stage's `full` barrier: no consumer waits on a global load.
//                                (A value never straddles its aligned word, so the word lies inside the allocation.)
//   warps 10, 11   idle        : they complete the producer warpgroup, see NTHREADS.
// Stage shared memory: activations (A_TILE), packed bytes (W_TILE), coefficient words [set][s_lo, s_hi, z_lo, z_hi][PR]
// (C_TILE; set 1 is the second group of a stage when the group size is 32).
// ------------------------------------------------------------------------------------------------
template <MmaKind KIND_, int T_, typename WT_, bool ZP_>
struct W4Cfg {
  static constexpr MmaKind KIND = KIND_;
  using WT = WT_;
  static constexpr bool ZP = ZP_;            // shift is an integer zero-point
  static constexpr int MWG = 2;              // consumer warpgroups
  static constexpr int T = T_;               // token rows per tile: the wgmma N
  static constexpr int NF = T == 256 ? 1 : 2;  // 64-row fragments (32 packed rows) per consumer warpgroup
  static constexpr int PR = 32 * NF * MWG;   // packed rows per tile
  static constexpr int A_TILE = T * 128;     // activations, [T][64 k]
  static constexpr int W_TILE = PR * 64;     // packed bytes, [PR][64 k]
  static constexpr int C_TILE = 2 * 4 * PR * 4;
  // output staging, one tile per 64 packed rows: two planes [T tokens][64 out-features]
  static constexpr int EPI_TILE = 2 * T * 128;
  static constexpr int EPI_BYTES = (PR / 64) * EPI_TILE;
  static constexpr int FIT = (220 * 1024 - EPI_BYTES) / (A_TILE + W_TILE + C_TILE);
  static constexpr int NSTAGES = FIT > 8 ? 8 : FIT;
  // full barrier: the TMA producer's arrive + the arrive-on of each lane of the coefficient warp
  using Pipe = PipeLayout<MWG, NSTAGES, A_TILE, W_TILE + C_TILE, 0, 33, EPI_BYTES>;
  // The producer side is a whole warpgroup (TMA warp, coefficient warp, two idle warps), so that registers can move
  // between warpgroups: each SM sub-partition's register file serves every fourth warp, and two consumer warpgroups
  // plus one producer warp would leave 168 registers per thread -- too few to keep 128 accumulators and the A
  // fragments of two steps, and ptxas would serialise the wgmmas.  The kernel launches at 168; with T >= 128 the
  // producer warpgroup gives back down to 56 and the consumers take 224 (64 accumulators need no more).
  // setmaxnreg.inc waits until the CTA's pool has the registers: the two must add up to what the CTA launched with.
  static constexpr int NTHREADS = (4 * MWG + 4) * 32;
  static constexpr int SMEM_BYTES = Pipe::SMEM_BYTES;
  static constexpr bool REALLOC = T >= 128;
  static constexpr int REG_CONSUMER = 224, REG_PRODUCER = 56;
  static_assert(!REALLOC || 128 * MWG * REG_CONSUMER + 128 * REG_PRODUCER <= ((65536 / NTHREADS) & ~7) * NTHREADS,
                "register reallocation exceeds the CTA's launch allocation");
  static_assert(T == 64 || T == 128 || T == 256, "token tile");
  static_assert(NSTAGES >= 4, "stage ring depth");
};

// Epilogue of the swap-AB kernel, the threads that share one staging tile (64 packed rows: one consumer warpgroup when
// NF = 2, both when NF = 1).  acc[f * T/2 + 4 j + 2 h + e] is out-feature row 32 fc + 8 w + g of the staging tile
// (fc = f, or wg when NF = 1) of nibble plane h (packed row n_pr0 + that; out-feature N/2 + that for h = 1), token
// 8 j + 2 c + e.  The rounded values go TRANSPOSED into the staging tile (two planes [T tokens][64 out-features],
// 128-byte rows, 128-byte swizzle) with stmatrix: each 8 x 8 block of the fragment becomes 8 token rows of one 16-byte
// chunk.  From there the tile leaves as in int4_epilogue: two TMA stores into [M, 2, N/2], or the ordinary
// bounds-checked copy-out.
template <typename OT, int T, int NF>
__device__ __forceinline__ void w4_epilogue(const GemmParams& p, const CUtensorMap* tmap_out,
                                            const float (&acc)[NF * T / 2], uint32_t stile, int row0, int n_pr0, int wg) {
  constexpr int PLANE = T * 128;
  constexpr int ET = NF == 1 ? 256 : 128;  // threads of the staging tile
  const int bar = NF == 1 ? 1 : 1 + wg;
  const int t = static_cast<int>(threadIdx.x) & (ET - 1);
  const int lane = t & 31, w = (t >> 5) & 3, g = lane >> 2;
  const int half_n = p.N / 2;
  const OT* bias = static_cast<const OT*>(p.bias);
  if (t == 0) bulk_wait_group_read<0>();
  named_bar_sync(bar, ET);
  // stmatrix addresses: lane 8 q + i names token row 8 (4 jj + q) + i of matrix q; (token % 8) == i
  const uint32_t i = static_cast<uint32_t>(lane) & 7;
  const uint32_t lane_row = stile + ((static_cast<uint32_t>(lane) >> 3) * 8 + i) * 128;
#pragma unroll
  for (int f = 0; f < NF; ++f) {
    const int fc = NF == 1 ? wg : f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = (h ? half_n : 0) + n_pr0 + 32 * fc + 8 * w + g;
      const float b = (bias != nullptr && n < (h ? p.N : half_n)) ? to_float<OT>(bias[n]) : 0.f;
      const uint32_t chunk = ((static_cast<uint32_t>(4 * fc + w) ^ i) << 4) + h * PLANE;
#pragma unroll
      for (int jj = 0; jj < T / 32; ++jj) {
        uint32_t r[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int j = 4 * jj + q;
          float f0 = acc[f * (T / 2) + 4 * j + 2 * h], f1 = acc[f * (T / 2) + 4 * j + 2 * h + 1];
          rnd_pair<OT>(f0, f1);
          if (bias != nullptr) {
            f0 = __fadd_rn(f0, b);
            f1 = __fadd_rn(f1, b);
            rnd_pair<OT>(f0, f1);
          }
          r[q] = pack2<OT>(f0, f1);
        }
        stmatrix_x4_trans(lane_row + jj * 32 * 128 + chunk, r[0], r[1], r[2], r[3]);
      }
    }
  }
  fence_proxy_async_smem();  // the tile's generic-proxy writes -> visible to the TMA store
  named_bar_sync(bar, ET);
  if (p.epi_tma) {
    if (t == 0 && row0 < p.M) {
      tma_store_3d(tmap_out, stile, n_pr0, 0, row0);
      tma_store_3d(tmap_out, stile + PLANE, n_pr0, 1, row0);
      bulk_commit_group();
    }
    return;
  }
  // copy-out: thread t moves column pair 2 (t % 64) of token rows t / 64, t / 64 + ET / 64, ...
  const int c = 2 * (t & 63);
  const int plane = c >> 6, pc = c & 63;
  const int n = (plane ? half_n : 0) + n_pr0 + pc;
  const int n_limit = plane ? p.N : half_n;
  if (n >= n_limit) return;
  const bool two = n + 1 < n_limit;
  const uint32_t src = stile + plane * PLANE + (pc & 7) * 2;
  for (int r = t >> 6; r < T && row0 + r < p.M; r += ET / 64) {
    const uint32_t v = ld_shared_u32(src + r * 128 + ((static_cast<uint32_t>(pc >> 3) ^ (r & 7)) << 4));
    const size_t off = static_cast<size_t>(row0 + r) * p.ld + p.col0 + n;
    const bool vec = (off * sizeof(OT)) % (2 * sizeof(OT)) == 0;
    for (int q = 0; q < p.g.n_out; ++q) {
      uint16_t* dst = static_cast<uint16_t*>(p.g.out_peer[q]) + off;
      if (two && vec) {
        *reinterpret_cast<uint32_t*>(dst) = v;
      } else {
        dst[0] = static_cast<uint16_t>(v);
        if (two) dst[1] = static_cast<uint16_t>(v >> 16);
      }
    }
  }
}

// the aligned 4-byte word that holds byte `off` of `base`, and the bit position of that byte in it
__device__ __forceinline__ const void* word_of(const void* base, size_t off) {
  return reinterpret_cast<const void*>((reinterpret_cast<uintptr_t>(base) + off) & ~static_cast<uintptr_t>(3));
}
__device__ __forceinline__ uint32_t bitpos_of(const void* base, size_t off) {
  return static_cast<uint32_t>((reinterpret_cast<uintptr_t>(base) + off) & 3) * 8;
}

// keeps the compiler from moving writes of a wgmma A fragment above the wgmma_wait that frees its registers
__device__ __forceinline__ void fence_frag(uint32_t (&a)[4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(a[i])::"memory");
}

template <class Cfg>
__global__ void __launch_bounds__(Cfg::NTHREADS, 1)
    gemm_w4_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_w,
                   const __grid_constant__ CUtensorMap tmap_out, const GemmParams p) {
  using L = typename Cfg::Pipe;
  using WT = typename Cfg::WT;
  using D = Dq<WT>;
  constexpr int T = Cfg::T, PR = Cfg::PR, NF = Cfg::NF;
  constexpr bool ZP = Cfg::ZP;

  const auto pipe = WgmmaPipe<L>::init([&] {
    tma_prefetch_desc(&tmap_a);
    tma_prefetch_desc(&tmap_w);
    if (p.epi_tma) tma_prefetch_desc(&tmap_out);
  });

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.num_m_blocks * p.num_n_blocks;
  const int kblocks = (p.K + 63) / 64;
  const int half_n = p.N / 2;
  const int gpr = p.K / p.group;       // groups per out-feature row
  const bool two_sets = p.group < 64;  // group size 32: two (scale, shift) sets per 64-k stage

  if (warp < L::PRODUCER_WARP) {
    // ------------------------------------------------------------------ consumers: dequantise + wgmma + epilogue
    if constexpr (Cfg::REALLOC) setmaxnreg_inc<Cfg::REG_CONSUMER>();
    const int wg = warp >> 2;
    const int g = lane >> 2, c = lane & 3;
    const int r0 = 32 * NF * wg + 8 * (warp & 3) + g;  // this thread's packed row of fragment 0 in the tile (+32: fragment 1)
    uint32_t roff[NF], rsw[NF];
#pragma unroll
    for (int f = 0; f < NF; ++f) {
      const uint32_t r = static_cast<uint32_t>(r0 + 32 * f);
      roff[f] = r * 64 + 4 * (static_cast<uint32_t>(c) >> 1);  // word c / 2 of a chunk holds k 2c, 2c+1; word 2 + c / 2 k 2c+8, 2c+9
      rsw[f] = (r >> 1) & 3;
    }
    const uint32_t sel = (c & 1) ? 0x7632u : 0x5410u;
    float acc[NF * T / 2];
    RingPos<L::NSTAGES> pos;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile % p.num_m_blocks;
      const int n_blk = tile / p.num_m_blocks;
      const int rp0 = n_blk * PR + r0;
      int kb = 0;
      // byte position (mod 4) of group 0 of s_lo, s_hi, z_lo, z_hi of fragment f's packed row inside its aligned word
      uint32_t cb[NF][4];
#pragma unroll
      for (int f = 0; f < NF; ++f) {
        const size_t ilo = static_cast<size_t>(rp0 + 32 * f) * gpr;
        const size_t ihi = ilo + static_cast<size_t>(half_n) * gpr;
        cb[f][0] = bitpos_of(p.wscale, 2 * ilo) >> 3;
        cb[f][1] = bitpos_of(p.wscale, 2 * ihi) >> 3;
        cb[f][2] = bitpos_of(p.wshift, (ZP ? 1 : 2) * ilo) >> 3;
        cb[f][3] = bitpos_of(p.wshift, (ZP ? 1 : 2) * ihi) >> 3;
      }
      // (scale, shift) of both nibbles of fragment f's packed row for coefficient set `set` of the stage at k `kset`
      auto coefs = [&](uint32_t ct, int set, int kset, typename D::Coef (&klo)[NF], typename D::Coef (&khi)[NF]) {
        const uint32_t grp = static_cast<uint32_t>((p.group_log2 >= 0) ? (kset >> p.group_log2) : (kset / p.group));
        const uint32_t gs = 2 * grp, gz = (ZP ? 1 : 2) * grp;
#pragma unroll
        for (int f = 0; f < NF; ++f) {
          const uint32_t a = ct + static_cast<uint32_t>(set * 4 * PR + r0 + 32 * f) * 4;
          const uint16_t s_lo = static_cast<uint16_t>(ld_shared_u32(a) >> (((cb[f][0] + gs) & 3) << 3));
          const uint16_t s_hi = static_cast<uint16_t>(ld_shared_u32(a + PR * 4) >> (((cb[f][1] + gs) & 3) << 3));
          uint16_t z_lo = static_cast<uint16_t>(ld_shared_u32(a + 2 * PR * 4) >> (((cb[f][2] + gz) & 3) << 3));
          uint16_t z_hi = static_cast<uint16_t>(ld_shared_u32(a + 3 * PR * 4) >> (((cb[f][3] + gz) & 3) << 3));
          if (ZP) {
            z_lo &= 0xFF;
            z_hi &= 0xFF;
          }
          klo[f] = D::make_raw(bits_as<WT>(s_lo), z_lo, ZP);
          khi[f] = D::make_raw(bits_as<WT>(s_hi), z_hi, ZP);
        }
      };
      pipe.consume_tile(pos, kblocks, acc, [&](uint32_t, uint32_t wt, bool accumulate) {
        const uint32_t act = wt - Cfg::A_TILE, ct = wt + Cfg::W_TILE;
        const int kbase = 64 * kb++;
        // steps 2 and 3 read set 1 with groups of 32, except in a K tail (K % 64 == 32) where their activations are zero
        // and set 0 stands in.  Otherwise the stage has one set and steps 2 and 3 keep the coefficients of step 0:
        // re-reading them put four shared loads and the coefficient arithmetic in front of step 2's wgmma (the branch is
        // uniform over the warpgroup, and ptxas keeps the wgmmas asynchronous).
        const bool set2 = two_sets && kbase + 32 < p.K;
        typename D::Coef klo[NF], khi[NF];
        coefs(ct, 0, kbase, klo, khi);
        uint32_t a[2][NF][4];  // [step parity][fragment]: the registers of the step in flight stay untouched
#pragma unroll
        for (int st = 0; st < 4; ++st) {
          if (st == 2 && set2) coefs(ct, 1, kbase + 32, klo, khi);
#pragma unroll
          for (int f = 0; f < NF; ++f) {
            uint32_t (&af)[4] = a[st & 1][f];
            fence_frag(af);
            const uint32_t chunk = wt + roff[f] + ((static_cast<uint32_t>(st) ^ rsw[f]) << 4);
            const uint32_t x = __byte_perm(ld_shared_u32(chunk), ld_shared_u32(chunk + 8), sel);
            if (QB_KO(p.dbg, 1)) {  // developer experiment: no dequantisation, the raw packed word as the A fragment
              af[0] = af[1] = af[2] = af[3] = x;
            } else {
              const uint32_t wl = x & 0x0F0F0F0Fu, wh = (x >> 4) & 0x0F0F0F0Fu;
              af[0] = D::cvt(__byte_perm(wl, D::MAGIC_BYTES, 0x4140), klo[f], ZP);  // row g,     k 2c, 2c+1
              af[1] = D::cvt(__byte_perm(wh, D::MAGIC_BYTES, 0x4140), khi[f], ZP);  // row g + 8, k 2c, 2c+1
              af[2] = D::cvt(__byte_perm(wl, D::MAGIC_BYTES, 0x4342), klo[f], ZP);  // row g,     k 2c+8, 2c+9
              af[3] = D::cvt(__byte_perm(wh, D::MAGIC_BYTES, 0x4342), khi[f], ZP);  // row g + 8, k 2c+8, 2c+9
            }
          }
          wgmma_fence();
          const uint64_t db = wgmma_desc_sw128(act + st * 32);
#pragma unroll
          for (int f = 0; f < NF; ++f)
            wgmma_rs<Cfg::KIND, T>(*reinterpret_cast<float(*)[T / 2]>(acc + f * (T / 2)), a[st & 1][f], db,
                                   (st > 0 || accumulate) ? 1u : 0u);
          // the last step is committed by consume_tile, whose wait retires step 2 before the next stage writes its set.
          // One step in flight: with wait_group 2 (and four A buffers at T = 256) ptxas serialises the wgmmas (C7513).
          if (st < 3) {
            wgmma_commit();
            wgmma_wait<1>();  // retires step st - 1: its registers take step st + 1
          }
        }
      });
      // the staging tile of this warpgroup's packed rows (both warpgroups share one when NF = 1)
      const int et = NF == 1 ? 0 : wg;
      w4_epilogue<WT, T, NF>(p, &tmap_out, acc, pipe.epi + et * Cfg::EPI_TILE, m_blk * T, n_blk * PR + 64 * et, wg);
    }
    if ((threadIdx.x & 127) == 0) bulk_wait_group_all();  // the last tile's TMA store has completed
    if (p.g.n_out > 1) __threadfence_system();            // this thread's peer stores are performed before the rank signals
  } else {
    if constexpr (Cfg::REALLOC) setmaxnreg_dec<Cfg::REG_PRODUCER>();
    if (warp == L::PRODUCER_WARP && lane == 0) {
      // ---------------------------------------------------------------- TMA producer: activations + packed bytes
      gather_wait_start(p.g);  // the activation may be the gathered output of the previous linear
      // developer experiment 8: no activation feed after the first NSTAGES k-blocks of a tile (the stages keep stale data)
      const bool no_act = QB_KO(p.dbg, 8);
      pipe.produce(num_tiles, p.num_m_blocks, kblocks, (no_act ? 0 : Cfg::A_TILE) + Cfg::W_TILE,
                   [&](uint8_t* dst, uint64_t* bar, int m_blk, int n_blk, int kb) {
                     if (!no_act || kb < L::NSTAGES) {
                       if (no_act) mbar_expect_tx(bar, Cfg::A_TILE);
                       tma_load_2d(dst, &tmap_a, bar, kb * 64, m_blk * T);
                     }
                     tma_load_2d(dst + Cfg::A_TILE, &tmap_w, bar, kb * 64, n_blk * PR);
                   });
    } else if (warp == L::PRODUCER_WARP + 1) {
      // ---------------------------------------------------------------- the stages' scales and shifts
      constexpr size_t ZB = ZP ? 1 : 2;  // bytes per shift
      const int nsets = two_sets ? 2 : 1;
      RingPos<L::NSTAGES> pos;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n_blk = tile / p.num_m_blocks;
        for (int kb = 0; kb < kblocks; ++kb) {
          mbar_wait(&pipe.empty_bar[pos.stage], pos.phase ^ 1u);
          const uint32_t ct = pipe.b_addr(pos.stage) + Cfg::W_TILE;
          const int kbase = 64 * kb;
          const int g0 = (p.group_log2 >= 0) ? (kbase >> p.group_log2) : (kbase / p.group);
          for (int e = lane; e < nsets * PR; e += 32) {
            const int set = e >= PR ? 1 : 0;
            const int row = e - set * PR;
            const int rp = n_blk * PR + row;
            // rows past N/2 are never stored; a K-tail second group (K % 64 == 32) is never read
            if (rp >= half_n || (set == 1 && kbase + 32 >= p.K) || QB_KO(p.dbg, 4)) continue;
            const size_t ilo = static_cast<size_t>(rp) * gpr + g0 + set;
            const size_t ihi = ilo + static_cast<size_t>(half_n) * gpr;
            const uint32_t d = ct + static_cast<uint32_t>(set * 4 * PR + row) * 4;
            cp_async_4(d, word_of(p.wscale, 2 * ilo));
            cp_async_4(d + PR * 4, word_of(p.wscale, 2 * ihi));
            cp_async_4(d + 2 * PR * 4, word_of(p.wshift, ZB * ilo));
            cp_async_4(d + 3 * PR * 4, word_of(p.wshift, ZB * ihi));
          }
          cp_async_mbar_arrive_noinc(smem_u32(&pipe.full_bar[pos.stage]));
          pos.advance();
        }
      }
    }
  }

  __syncthreads();
  if (threadIdx.x == 0) gather_signal_end(p.g);  // fused all-gather: publish "this rank's slab has landed everywhere"
}

// ------------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------------
// Parameters of a problem with one dense [M, N] output of `out_dt` elements (g.n_out = 1, ld = N, col0 = 0); every
// other field zero.
inline GemmParams dense_gemm_params(void* out, const void* bias, int out_dt, int64_t m, int64_t n, int64_t k) {
  GemmParams p{};
  p.bias = bias;
  p.out = out;
  p.g.out_peer[0] = out;
  p.g.n_out = 1;
  p.g.world = 1;
  p.ld = static_cast<int>(n);
  p.col0 = 0;
  p.out_dt = out_dt;
  p.M = static_cast<int>(m);
  p.N = static_cast<int>(n);
  p.K = static_cast<int>(k);
  return p;
}

// Launch gemm_tc_kernel<Cfg> over p's tiles.  A null tensor map is passed zeroed: the operand the kernel's own warps
// stage (the weights of INT4 / BYTES, both operands of F8) and the output of every epilogue but the int4 TMA store.
template <class Cfg>
int launch_gemm_tc(const CUtensorMap* ta, const CUtensorMap* tb, const CUtensorMap* tout, const GemmParams& p,
                   cudaStream_t stream, const char* what = "gemm_tc_kernel launch") {
  const CUtensorMap zero{};
  return launch_persistent<gemm_tc_kernel<Cfg>, typename Cfg::Pipe>(p.num_m_blocks * p.num_n_blocks, stream, what,
                                                                    ta ? *ta : zero, tb ? *tb : zero,
                                                                    tout ? *tout : zero, p);
}

}  // namespace qb
