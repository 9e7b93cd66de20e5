// Persistent, warp-specialised wgmma kernel for the input gradient of the quantized linear (Hopper, sm_90a):
//
//   dX[m, k] = sum_n gO[m, n] * dequant(W)[n, k]
//
// One CTA per SM loops over BM x 128 tiles of dX (BM = 64 per consumer warpgroup); the columns of a tile are the weight's
// in-features k and the reduction runs over its out-features n.  The pipeline is the forward's (wgmma_pipe.cuh); roles:
//   warps [0, 4*MWG)  consumers    : wgmma with fp32 accumulators in registers, then one rounding to the gradient dtype
//   warp 4*MWG        TMA producer : the gO tiles
//   further warps     staging      : read the packed int4 (or 8-bit) weight bytes, dequantise them with the forward's exact
//                                    rounding (Dq / dequant16, cvt_bytes4: the operands are bit-identical to
//                                    qb200_dequantize_qbits / the reference's QBytesDequantizer) and write the tile
//
// Shared-memory layout of one stage:
//   A (gO, K-major, written by TMA with SWIZZLE_128B): BM rows x 64 reduction indices (128 bytes), one tile per plane.
//   B (weight, MN-major): one row of 128 k (256 bytes) per reduction index n, split into two swizzle atoms of 64 k;
//     row r of an atom lives at (r/8)*1024 + (r%8)*128 and its 16-byte chunk c at chunk position c ^ (r%8).
//
// int4 (canonical packing, [N/2, K] bytes, low nibble = n, high nibble = n + N/2): a stage is 64 packed rows
// [p0, p0 + 64) and holds 128 reduction indices, n = p0 + i (B rows 0..63, low nibbles) and N/2 + p0 + i (B rows 64..127,
// high nibbles).  gO is described as a 3-D tensor [M, 2, N/2] so that the two A boxes of a stage (columns p0 + i and
// N/2 + p0 + i) never cross N/2: TMA zero-fills the reduction tail of each plane instead of reading the other plane.
// 8-bit weights ([N, K], per-row scale): a stage is 64 reduction rows and one A box of a 2-D [M, N] description.
#pragma once

#include "gemm_tc.cuh"

namespace qb {

struct DgradParams {
  void* out;           // dX [M, K] in WT
  const uint8_t* w;    // int4: packed [N/2, K] bytes ; 8-bit: W [N, K]
  const void* wscale;  // int4: [N * K / group] ; 8-bit: [N]   (WT)
  const void* wshift;  // int4 only: [N * K / group], WT or uint8 zero-points
  int M, N, K;
  int group, group_log2;
  int num_m_blocks, num_k_blocks;  // output tiles
  int red_blocks;                  // pipeline stages per tile (reduction)
};

// INT4_: packed int4 weights (else 8-bit, WKIND_ as in GemmCfg).  MWG_: consumer warpgroups (BM = 64 * MWG_).
template <bool INT4_, int MWG_, typename WT_, bool ZP_ = false, int WKIND_ = 0>
struct DgradCfg {
  static constexpr bool INT4 = INT4_;
  static constexpr int MWG = MWG_;
  static constexpr int BM = 64 * MWG;
  static constexpr bool ZP = ZP_;
  static constexpr int WKIND = WKIND_;
  using WT = WT_;
  static constexpr MmaKind KIND = std::is_same<WT, __half>::value ? MmaKind::F16 : MmaKind::BF16;
  static constexpr int BN = 128;                        // dX columns per tile
  static constexpr int RED = INT4 ? 128 : 64;           // reduction indices per stage
  static constexpr int A_PLANE = BM * 128;              // one [BM, 64] box of gO
  static constexpr int A_TILE = (INT4 ? 2 : 1) * A_PLANE;
  static constexpr int B_ATOM = RED * 128;              // 64 k columns of every reduction row of the stage
  static constexpr int B_TILE = 2 * B_ATOM;
  static constexpr int NSTAGES = 3;
  // 64 staging threads per slot: one packed (or 8-bit) row each; the TMA producer's arrive for gO
  using Pipe = PipeLayout<MWG, NSTAGES, A_TILE, B_TILE, 2, 1>;
};

template <class Cfg>
__global__ void __launch_bounds__(Cfg::Pipe::NTHREADS, 1)
    gemm_dgrad_kernel(const __grid_constant__ CUtensorMap tmap_g, const DgradParams p) {
  using L = typename Cfg::Pipe;
  using WT = typename Cfg::WT;

  const auto pipe = WgmmaPipe<L>::init([&] { tma_prefetch_desc(&tmap_g); });

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int num_tiles = p.num_m_blocks * p.num_k_blocks;
  const int kblocks = p.red_blocks;

  if (warp < L::PRODUCER_WARP) {
    // ------------------------------------------------------------------ consumers: wgmma + epilogue
    const int wg = warp >> 2;
    float acc[64];
    RingPos<L::NSTAGES> pos;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile % p.num_m_blocks;
      const int k_blk = tile / p.num_m_blocks;
      pipe.consume_tile(pos, kblocks, acc, [&](uint32_t aa, uint32_t bb, bool accumulate) {
#pragma unroll
        for (int s = 0; s < Cfg::RED / 16; ++s) {
          // int4: steps 0..3 reduce the low-nibble plane (A box 0), steps 4..7 the high-nibble plane (A box 1)
          const uint32_t a_s = aa + (s / 4) * Cfg::A_PLANE + (s % 4) * 32;
          const uint32_t b_s = bb + s * 2048;  // 16 reduction rows = two 8-row groups
          wgmma_n128_tb<Cfg::KIND>(acc, wgmma_desc_sw128(a_s), wgmma_desc_sw128_mn(b_s, Cfg::B_ATOM),
                                   (s > 0 || accumulate) ? 1u : 0u);
        }
      });
      // fragment: thread holds rows r0 and r0 + 8, column pairs 8 j + 2 (lane % 4); K % 16 == 0, so a pair is whole
      const int r0 = m_blk * Cfg::BM + wg * 64 + (warp & 3) * 16 + (lane >> 2);
      WT* out = static_cast<WT*>(p.out);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        if (row >= p.M) continue;
        WT* orow = out + static_cast<size_t>(row) * p.K;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int k = k_blk * 128 + 8 * j + 2 * (lane & 3);
          if (k >= p.K) continue;
          *reinterpret_cast<uint32_t*>(orow + k) = pack2<WT>(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      }
    }
  } else if (warp == L::PRODUCER_WARP) {
    // ------------------------------------------------------------------ TMA producer (gO)
    if (lane == 0) {
      pipe.produce(num_tiles, p.num_m_blocks, kblocks, Cfg::A_TILE, [&](uint8_t* dst, uint64_t* bar, int m_blk, int, int kb) {
        if constexpr (Cfg::INT4) {
          tma_load_3d(dst, &tmap_g, bar, kb * 64, 0, m_blk * Cfg::BM);
          tma_load_3d(dst + Cfg::A_PLANE, &tmap_g, bar, kb * 64, 1, m_blk * Cfg::BM);
        } else {
          tma_load_2d(dst, &tmap_g, bar, kb * 64, m_blk * Cfg::BM);
        }
      });
    }
  } else {
    // ------------------------------------------------------------------ weight staging
    StagingThread<L> sg(pipe, num_tiles, kblocks);
    const int r = sg.r;
    const uint32_t sw = static_cast<uint32_t>(r) & 7;
    const uint32_t off_r = (static_cast<uint32_t>(r) >> 3) * 1024 + (static_cast<uint32_t>(r) & 7) * 128;

    if constexpr (Cfg::INT4) {
      using D = Dq<WT>;
      constexpr bool ZP = Cfg::ZP;
      const int half_n = p.N / 2;
      const int gpr = p.K / p.group;  // groups per out-feature
      // A stage covers 128 k: at most 4 groups (group 32), else at most 2.  Coefficient set `st` is group g0 + st,
      // clamped to the row's last group so that the columns past K never read past the scale / shift arrays.
      struct Pre {
        uint4 raw[8];
        uint32_t s[4], z[4];  // low plane in bits [0, 16), high plane in [16, 32)
        int k0, g0;
        bool ok = false;
      };
      auto load_pre = [&](Pre& pr, const StageSeq<L::NSTAGES>& seq) {
        const int rp = seq.kb * 64 + r;
        const int k0 = (seq.tile / p.num_m_blocks) * 128;
        pr.k0 = k0;
        pr.ok = rp < half_n;
        if (pr.ok) {
          const uint8_t* src = p.w + static_cast<size_t>(rp) * p.K + k0;
#pragma unroll
          for (int v = 0; v < 8; ++v)
            pr.raw[v] = (k0 + v * 16 < p.K) ? __ldg(reinterpret_cast<const uint4*>(src + v * 16)) : make_uint4(0, 0, 0, 0);
          const int g0 = (p.group_log2 >= 0) ? (k0 >> p.group_log2) : (k0 / p.group);
          pr.g0 = g0;
          const size_t row_lo = static_cast<size_t>(rp) * gpr, row_hi = row_lo + static_cast<size_t>(half_n) * gpr;
          pr.s[2] = pr.s[3] = pr.z[2] = pr.z[3] = 0u;
#pragma unroll
          for (int st = 0; st < 4; ++st) {
            if (st > 1 && p.group >= 64) break;  // groups of 64 or more span at most two sets of a 128-k stage
            const int g = min(g0 + st, gpr - 1);
            const CoefPair c = load_coef_pair<ZP>(p.wscale, p.wshift, row_lo + g, row_hi + g);
            pr.s[st] = c.s_lo | (static_cast<uint32_t>(c.s_hi) << 16);
            pr.z[st] = c.z_lo | (static_cast<uint32_t>(c.z_hi) << 16);
          }
        }
      };
      sg.template run_ping_pong<Pre>(load_pre, [&](const Pre& cur) {
        sg.wait_empty();
        if (cur.ok) {
#pragma unroll
          for (int v = 0; v < 8; ++v) {
            // coefficient set of this 16-k chunk: its group minus the stage's first group (past K: clamped)
            const int kv = cur.k0 + v * 16;
            int gv = (p.group_log2 >= 0) ? (kv >> p.group_log2) : (kv / p.group);
            int st = gv - cur.g0;
            st = st > 3 ? 3 : st;
            const uint32_t s = st == 0 ? cur.s[0] : (st == 1 ? cur.s[1] : (st == 2 ? cur.s[2] : cur.s[3]));
            const uint32_t z = st == 0 ? cur.z[0] : (st == 1 ? cur.z[1] : (st == 2 ? cur.z[2] : cur.z[3]));
            const typename D::Coef klo = D::make_raw(bits_as<WT>(static_cast<uint16_t>(s & 0xFFFFu)),
                                                     static_cast<uint16_t>(z & 0xFFFFu), ZP);
            const typename D::Coef khi = D::make_raw(bits_as<WT>(static_cast<uint16_t>(s >> 16)),
                                                     static_cast<uint16_t>(z >> 16), ZP);
            uint32_t lo[8], hi[8];
            dequant16<WT, ZP>(cur.raw[v], klo, khi, lo, hi);
            const uint32_t atom = sg.bt + (v / 4) * Cfg::B_ATOM + off_r;
            const uint32_t c0 = ((2u * (v % 4) + 0u) ^ sw) << 4, c1 = ((2u * (v % 4) + 1u) ^ sw) << 4;
            constexpr uint32_t HI = 8 * 1024;  // B rows 64..127: the high-nibble plane
            st_shared_v4(atom + c0, lo[0], lo[1], lo[2], lo[3]);
            st_shared_v4(atom + c1, lo[4], lo[5], lo[6], lo[7]);
            st_shared_v4(atom + HI + c0, hi[0], hi[1], hi[2], hi[3]);
            st_shared_v4(atom + HI + c1, hi[4], hi[5], hi[6], hi[7]);
          }
        } else {
#pragma unroll
          for (int a = 0; a < 2; ++a)
#pragma unroll
            for (int c = 0; c < 8; ++c) {
              st_shared_v4(sg.bt + a * Cfg::B_ATOM + off_r + (c << 4), 0u, 0u, 0u, 0u);
              st_shared_v4(sg.bt + a * Cfg::B_ATOM + off_r + 8 * 1024 + (c << 4), 0u, 0u, 0u, 0u);
            }
        }
        sg.publish();
      });
    } else {
      // ---------------- 8-bit weights: thread r converts reduction row n = kb * 64 + r, rnd(scale[n] * W[n, k])
      struct PreB {
        uint4 raw[8];
        uint32_t s2;
      };
      const WT* scale = static_cast<const WT*>(p.wscale);
      auto load_pre = [&](PreB& pr, const StageSeq<L::NSTAGES>& seq) {
        const int n = seq.kb * 64 + r;
        const int k0 = (seq.tile / p.num_m_blocks) * 128;
        const bool ok = n < p.N;
        const uint8_t* src = p.w + static_cast<size_t>(ok ? n : 0) * p.K + k0;
#pragma unroll
        for (int v = 0; v < 8; ++v)
          pr.raw[v] = (ok && k0 + v * 16 < p.K) ? __ldg(reinterpret_cast<const uint4*>(src + v * 16)) : make_uint4(0, 0, 0, 0);
        // rows past N: zero bytes times a zero scale -> exact zeros (their gO columns are zero-filled as well)
        const WT sv = ok ? scale[n] : from_float<WT>(0.f);
        pr.s2 = static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(&sv)) * 0x00010001u;
      };
      sg.template run_ping_pong<PreB>(load_pre, [&](const PreB& cur) {
        sg.wait_empty();
#pragma unroll
        for (int v = 0; v < 8; ++v) {
          uint32_t o[8];
          cvt_bytes4<WT, Cfg::WKIND>(cur.raw[v].x, cur.s2, o[0], o[1]);
          cvt_bytes4<WT, Cfg::WKIND>(cur.raw[v].y, cur.s2, o[2], o[3]);
          cvt_bytes4<WT, Cfg::WKIND>(cur.raw[v].z, cur.s2, o[4], o[5]);
          cvt_bytes4<WT, Cfg::WKIND>(cur.raw[v].w, cur.s2, o[6], o[7]);
          const uint32_t atom = sg.bt + (v / 4) * Cfg::B_ATOM + off_r;
          st_shared_v4(atom + (((2u * (v % 4) + 0u) ^ sw) << 4), o[0], o[1], o[2], o[3]);
          st_shared_v4(atom + (((2u * (v % 4) + 1u) ^ sw) << 4), o[4], o[5], o[6], o[7]);
        }
        sg.publish();
      });
    }
  }
}

}  // namespace qb
