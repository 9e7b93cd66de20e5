// Very-small-M (M <= 32, "batch 1..32 decode") fused packed-int4 linear as a pure streaming kernel.
//
// This path is HBM-bound: what matters is that every SM keeps many 128-bit loads of packed weight bytes in flight and
// spends as few issue slots per weight as the exact dequantisation allows.  So there is no shared-memory staging, no
// TMA ring and no tensor-memory round trip here: each thread loads the packed bytes of "its" out-features straight
// into registers (coalesced LDG.128, 4 lanes cover 64 contiguous bytes of a packed row), dequantises them in
// registers with the reference's rounding order, and feeds them as the A fragment of a warp-level
// mma.sync.m16n8k16 (16 out-features x 8 tokens per instruction) whose B fragment is the activation vector.
// The k index of an MMA is only a summation index, so the k positions are permuted to what the loads deliver
// (thread t of a quad owns k = 16t..16t+15 of each 64-k slab, k-step s uses its bytes 4s..4s+3) and the activation
// fragment is gathered with the same permutation.  The warp MMA is used on purpose: at <= 32 tokens the math is
// <2 % of the tensor peak, and unlike wgmma it takes its operands from registers, which is where the exact
// dequantisation leaves them.
//
// Decomposition (stream-K): blocks of 64 packed rows = 128 out-features, stages of 128 k; the P*K/128 stages are dealt
// to the CTAs in equal contiguous spans, so every SM streams the same number of bytes whatever N is.  A span is cut
// into segments at block boundaries; a block finished by several CTAs is reduced deterministically: every segment
// writes its fp32 partial to the workspace, an atomic ticket per block elects the last arriver, which sums the
// partials in segment order, rounds once, adds the bias and stores.  CTA = 8 warps: warp w handles the 16 packed rows
// (w & 3) of the block and the 64-k half (w >> 2) of every stage.
#pragma once

#include "common.cuh"
#include "gather.cuh"
#include "gemm_tc.cuh"

namespace qb {

struct DecodeParams {
  const void* scale;   // [N * K / group] weight dtype
  const void* shift;   // same, or uint8 zero-points
  const void* bias;    // [N] or nullptr
  void* out;           // [M, ld] (ld = N, col0 = 0 for an ordinary call)
  GatherInfo g;        // fused all-gather of a column-parallel linear (gather.cuh); g.n_out == 1: ordinary call
  int ld, col0;
  float* partials;     // workspace: [P][max_segs][M][128] fp32
  int* tickets;        // workspace: [P] zero-initialised once; the kernel leaves them zero
  int M, N, K;
  int group;
  int group_log2;      // log2(group) or -1
  int shift_is_int;
  int P;               // out-feature blocks = ceil((N/2) / 64)
  int SPB;             // 128-k stages per block = K / 128
  int span;            // stages per CTA
  int max_segs;
  int dbg;             // developer knock-out flags (KNOCKOUTS=1 builds only)
};

// number of segments block `pb` is cut into when spans have `span` stages
__device__ __forceinline__ int decode_nsegs(int pb, int spb, int span) {
  return ((pb + 1) * spb - 1) / span - (pb * spb) / span + 1;
}

template <typename WT>
__device__ __forceinline__ void mma_m16n8k16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1);

template <>
__device__ __forceinline__ void mma_m16n8k16<__nv_bfloat16>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0,
                                                            uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
template <>
__device__ __forceinline__ void mma_m16n8k16<__half>(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

constexpr int kGemvThreads = 256;

// MT = ceil(M / 8) token tiles (1, 2 or 4)
template <typename WT, int MT, bool ZP>
__global__ void __launch_bounds__(kGemvThreads, (MT <= 2) ? 3 : 2)
    gemv_w4_kernel(const uint8_t* __restrict__ wq, const WT* __restrict__ x, const DecodeParams p) {
  using D = Dq<WT>;
  __shared__ float red[2][8 * MT][128];  // [k-half][token][tile row]   (8..32 KB)
  __shared__ int ticket_smem;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rb = warp & 3;   // 16-packed-row sub-block of the 64-row block
  const int kh = warp >> 2;  // which 64-k half of each 128-k stage
  const int g = lane >> 2;   // MMA row group: packed rows rb*16 + g and + 8 ; also the token column of the B fragment
  const int t = lane & 3;    // quad lane: owns k = 16t .. 16t+15 of the 64-k half
  const int half_n = p.N / 2;
  const int groups_per_row = p.K / p.group;
  const WT* scale = static_cast<const WT*>(p.scale);

  const int total = p.P * p.SPB;
  const int s_begin = min(static_cast<int>(blockIdx.x) * p.span, total);
  const int s_end = min(s_begin + p.span, total);
  const int L = s_end - s_begin;
  if (L <= 0) return;

  // ---- software prefetch ring (PF stages ahead): 2 x 16 packed bytes per thread and stage
  constexpr int PF = 4;
  uint4 w0[PF], w1[PF];  // packed rows r0 = rb*16+g and r0 + 8, bytes [k0 + kh*64 + 16t, +16)
  int f_i = 0;
  int f_pb = s_begin / p.SPB;
  int f_ks = s_begin - f_pb * p.SPB;
  auto fetch = [&](uint4& a, uint4& b) {
    if (f_i < L) {
      const int rp = f_pb * 64 + rb * 16 + g;
      const size_t off = static_cast<size_t>(f_ks) * 128 + kh * 64 + t * 16;
      a = (rp < half_n) ? __ldcs(reinterpret_cast<const uint4*>(wq + static_cast<size_t>(rp) * p.K + off))
                        : make_uint4(0, 0, 0, 0);
      b = (rp + 8 < half_n) ? __ldcs(reinterpret_cast<const uint4*>(wq + static_cast<size_t>(rp + 8) * p.K + off))
                            : make_uint4(0, 0, 0, 0);
      ++f_i;
      if (++f_ks == p.SPB) { f_ks = 0; ++f_pb; }
    }
  };
#pragma unroll
  for (int u = 0; u < PF - 1; ++u) fetch(w0[u], w1[u]);

  float acc_lo[MT][4], acc_hi[MT][4];
  auto zero_acc = [&]() {
#pragma unroll
    for (int m = 0; m < MT; ++m)
#pragma unroll
      for (int j = 0; j < 4; ++j) { acc_lo[m][j] = 0.f; acc_hi[m][j] = 0.f; }
  };
  zero_acc();

  int pb = s_begin / p.SPB, ks = s_begin - pb * p.SPB;
  for (int i0 = 0; i0 < L; i0 += PF) {
#pragma unroll
    for (int u = 0; u < PF; ++u) {
      const int i = i0 + u;
      if (i < L) {
        fetch(w0[(u + PF - 1) % PF], w1[(u + PF - 1) % PF]);
        // ---- per-stage coefficients of the four out-features this thread dequantises
        const int rp = pb * 64 + rb * 16 + g;
        const int k0 = ks * 128 + kh * 64;  // first k of this warp's 64-k half
        const bool ok0 = rp < half_n, ok1 = rp + 8 < half_n;
        // (scale, shift) may change every 32 k when group == 32: the thread's 16 k live in one group (group % 16 == 0)
        const int kk = k0 + t * 16;
        const int gi = (p.group_log2 >= 0) ? (kk >> p.group_log2) : (kk / p.group);
        typename D::Coef c_lo0, c_lo1, c_hi0, c_hi1;  // rows rp, rp+8 (low nibble) ; N/2+rp, N/2+rp+8 (high nibble)
        if (QB_KO(p.dbg, 4)) {  // developer experiment: no scale / shift traffic
          c_lo0 = c_lo1 = c_hi0 = c_hi1 = D::make_raw(from_float<WT>(0.01f), 0x3dcc, ZP);
        } else {
          const size_t i_lo0 = static_cast<size_t>(ok0 ? rp : 0) * groups_per_row + gi;
          const size_t i_lo1 = static_cast<size_t>(ok1 ? rp + 8 : 0) * groups_per_row + gi;
          const size_t hofs = static_cast<size_t>(half_n) * groups_per_row;
          c_lo0 = D::make(__ldg(scale + i_lo0), p.shift, i_lo0, ZP);
          c_lo1 = D::make(__ldg(scale + i_lo1), p.shift, i_lo1, ZP);
          c_hi0 = D::make(__ldg(scale + i_lo0 + hofs), p.shift, i_lo0 + hofs, ZP);
          c_hi1 = D::make(__ldg(scale + i_lo1 + hofs), p.shift, i_lo1 + hofs, ZP);
        }
        const uint32_t wa[4] = {w0[u].x, w0[u].y, w0[u].z, w0[u].w};
        const uint32_t wb[4] = {w1[u].x, w1[u].y, w1[u].z, w1[u].w};
#pragma unroll
        for (int s = 0; s < 4; ++s) {  // k-step s: this thread's k = kk + 4s .. +3
          uint32_t a_lo[4], a_hi[4];
          if (QB_KO(p.dbg, 1)) {  // developer experiment: no dequant arithmetic
            a_lo[0] = wa[s]; a_lo[1] = wb[s]; a_lo[2] = wa[s] >> 1; a_lo[3] = wb[s] >> 1;
            a_hi[0] = wa[s] >> 2; a_hi[1] = wb[s] >> 2; a_hi[2] = wa[s] >> 3; a_hi[3] = wb[s] >> 3;
          } else {
            const uint32_t l0 = wa[s] & 0x0F0F0F0Fu, h0 = (wa[s] >> 4) & 0x0F0F0F0Fu;
            const uint32_t l1 = wb[s] & 0x0F0F0F0Fu, h1 = (wb[s] >> 4) & 0x0F0F0F0Fu;
            a_lo[0] = D::cvt(__byte_perm(l0, D::MAGIC_BYTES, 0x4140), c_lo0, ZP);  // row g   , k slots 2t,2t+1
            a_lo[1] = D::cvt(__byte_perm(l1, D::MAGIC_BYTES, 0x4140), c_lo1, ZP);  // row g+8
            a_lo[2] = D::cvt(__byte_perm(l0, D::MAGIC_BYTES, 0x4342), c_lo0, ZP);  // row g   , k slots 2t+8,2t+9
            a_lo[3] = D::cvt(__byte_perm(l1, D::MAGIC_BYTES, 0x4342), c_lo1, ZP);
            a_hi[0] = D::cvt(__byte_perm(h0, D::MAGIC_BYTES, 0x4140), c_hi0, ZP);
            a_hi[1] = D::cvt(__byte_perm(h1, D::MAGIC_BYTES, 0x4140), c_hi1, ZP);
            a_hi[2] = D::cvt(__byte_perm(h0, D::MAGIC_BYTES, 0x4342), c_hi0, ZP);
            a_hi[3] = D::cvt(__byte_perm(h1, D::MAGIC_BYTES, 0x4342), c_hi1, ZP);
            if (!ok0) { a_lo[0] = a_lo[2] = a_hi[0] = a_hi[2] = 0u; }
            if (!ok1) { a_lo[1] = a_lo[3] = a_hi[1] = a_hi[3] = 0u; }
          }
#pragma unroll
          for (int m = 0; m < MT; ++m) {
            const int tok = m * 8 + g;
            uint2 xb = make_uint2(0u, 0u);
            if (tok < p.M && !QB_KO(p.dbg, 8))
              xb = __ldg(reinterpret_cast<const uint2*>(x + static_cast<size_t>(tok) * p.K + kk + 4 * s));
            if (QB_KO(p.dbg, 2)) {  // developer experiment: no tensor-core instruction
              acc_lo[m][0] += __uint_as_float(a_lo[0] ^ a_lo[1] ^ a_lo[2] ^ a_lo[3] ^ xb.x);
              acc_hi[m][0] += __uint_as_float(a_hi[0] ^ a_hi[1] ^ a_hi[2] ^ a_hi[3] ^ xb.y);
            } else {
              mma_m16n8k16<WT>(acc_lo[m], a_lo, xb.x, xb.y);
              mma_m16n8k16<WT>(acc_hi[m], a_hi, xb.x, xb.y);
            }
          }
        }

        // ---- segment end: reduce the two k-halves through shared memory, then the usual split-K fix-up
        const bool seg_end = ((ks == p.SPB - 1) || (i == L - 1)) && !QB_KO(p.dbg, 16);
        if (seg_end) {
#pragma unroll
          for (int m = 0; m < MT; ++m) {
            // D fragment: d0,d1 = (row g, tokens 2t,2t+1) ; d2,d3 = (row g+8, tokens 2t, 2t+1)
            const int r0 = rb * 16 + g;
            red[kh][m * 8 + 2 * t + 0][r0] = acc_lo[m][0];
            red[kh][m * 8 + 2 * t + 1][r0] = acc_lo[m][1];
            red[kh][m * 8 + 2 * t + 0][r0 + 8] = acc_lo[m][2];
            red[kh][m * 8 + 2 * t + 1][r0 + 8] = acc_lo[m][3];
            red[kh][m * 8 + 2 * t + 0][64 + r0] = acc_hi[m][0];
            red[kh][m * 8 + 2 * t + 1][64 + r0] = acc_hi[m][1];
            red[kh][m * 8 + 2 * t + 0][64 + r0 + 8] = acc_hi[m][2];
            red[kh][m * 8 + 2 * t + 1][64 + r0 + 8] = acc_hi[m][3];
          }
          zero_acc();
          __syncthreads();
          const int nsegs = decode_nsegs(pb, p.SPB, p.span);
          const int seg_idx = static_cast<int>(blockIdx.x) - (pb * p.SPB) / p.span;
          const int et = threadIdx.x;  // threads 0..127 own one tile row each
          const int rpe = pb * 64 + (et & 63);
          const bool n_ok = (et < 128) && rpe < half_n;
          const int n = (et < 64) ? rpe : half_n + rpe;
          if (et < 128) {
            if (nsegs == 1) {
              for (int m = 0; m < p.M; ++m) {
                if (n_ok) {
                  WT r = from_float<WT>(red[0][m][et] + red[1][m][et]);
                  if (p.bias != nullptr)
                    r = from_float<WT>(__fadd_rn(to_float<WT>(r), to_float<WT>(static_cast<const WT*>(p.bias)[n])));
                  static_cast<WT*>(p.out)[static_cast<size_t>(m) * p.N + n] = r;
                }
              }
            } else {
              float* part = p.partials + (static_cast<size_t>(pb) * p.max_segs + seg_idx) * p.M * 128;
              for (int m = 0; m < p.M; ++m) part[static_cast<size_t>(m) * 128 + et] = red[0][m][et] + red[1][m][et];
              asm volatile("fence.acq_rel.gpu;" ::: "memory");
            }
          }
          if (nsegs > 1) {
            __syncthreads();
            if (threadIdx.x == 0) {
              int tk;
              asm volatile("atom.acq_rel.gpu.global.add.s32 %0, [%1], 1;" : "=r"(tk) : "l"(p.tickets + pb) : "memory");
              ticket_smem = tk;
            }
            __syncthreads();
            if (ticket_smem == nsegs - 1 && et < 128) {
              asm volatile("fence.acq_rel.gpu;" ::: "memory");
              const float* base = p.partials + static_cast<size_t>(pb) * p.max_segs * p.M * 128 + et;
              for (int m = 0; m < p.M; ++m) {
                float sum = 0.f;
                for (int sg0 = 0; sg0 < nsegs; sg0 += 8) {
                  float v[8];
#pragma unroll
                  for (int b = 0; b < 8; ++b)
                    v[b] = (sg0 + b < nsegs) ? __ldcg(base + (static_cast<size_t>(sg0 + b) * p.M + m) * 128) : 0.f;
#pragma unroll
                  for (int b = 0; b < 8; ++b)
                    if (sg0 + b < nsegs) sum += v[b];
                }
                if (n_ok) {
                  WT r = from_float<WT>(sum);
                  if (p.bias != nullptr)
                    r = from_float<WT>(__fadd_rn(to_float<WT>(r), to_float<WT>(static_cast<const WT*>(p.bias)[n])));
                  static_cast<WT*>(p.out)[static_cast<size_t>(m) * p.N + n] = r;
                }
              }
              if (threadIdx.x == 0) p.tickets[pb] = 0;
            }
          }
          __syncthreads();  // `red` and `ticket_smem` are reused by the next segment
        }
        if (++ks == p.SPB) { ks = 0; ++pb; }
      }
    }
  }
}

}  // namespace qb
