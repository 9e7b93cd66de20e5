// Persistent, warp-specialised wgmma kernel for the input gradient of the quantized linear (Hopper, sm_90a):
//
//   dX[m, k] = sum_n gO[m, n] * dequant(W)[n, k]
//
// One CTA per SM loops over BM x 128 tiles of dX (BM = 64 per consumer warpgroup); the columns of a tile are the weight's
// in-features k and the reduction runs over its out-features n.  Roles, as in gemm_tc_kernel:
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
  static constexpr int STAGE = A_TILE + B_TILE;
  static constexpr int NSTAGES = 3;
  static constexpr int CVT_GROUP_WARPS = 2;             // 64 staging threads: one packed (or 8-bit) row each
  static constexpr int NCVT_WARPS = NSTAGES * CVT_GROUP_WARPS;
  static constexpr int PRODUCER_WARP = 4 * MWG;
  static constexpr int FIRST_CVT_WARP = PRODUCER_WARP + 1;
  static constexpr int NTHREADS = (FIRST_CVT_WARP + NCVT_WARPS) * 32;
  static constexpr int FULL_ARRIVALS = 1 + CVT_GROUP_WARPS;
  static constexpr int SMEM_BYTES = 1024 + NSTAGES * STAGE + 2 * NSTAGES * 8;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
};

template <typename WT>
__device__ __forceinline__ WT bits_as(uint16_t b) {
  return *reinterpret_cast<const WT*>(&b);
}

template <class Cfg>
__global__ void __launch_bounds__(Cfg::NTHREADS, 1)
    gemm_dgrad_kernel(const __grid_constant__ CUtensorMap tmap_g, const DgradParams p) {
  constexpr int NSTAGES = Cfg::NSTAGES;
  using WT = typename Cfg::WT;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + NSTAGES * Cfg::STAGE);
  uint64_t* empty_bar = full_bar + NSTAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == Cfg::PRODUCER_WARP * 32) {
    tma_prefetch_desc(&tmap_g);
    for (int s = 0; s < NSTAGES; ++s) {
      mbar_init(&full_bar[s], Cfg::FULL_ARRIVALS);
      mbar_init(&empty_bar[s], Cfg::MWG);
    }
    fence_mbar_init();
  }
  __syncthreads();

  const int num_tiles = p.num_m_blocks * p.num_k_blocks;
  const int kblocks = p.red_blocks;
  const uint32_t smem_base = smem_u32(smem);
  auto a_addr = [&](int s) { return smem_base + s * Cfg::STAGE; };
  auto b_addr = [&](int s) { return smem_base + s * Cfg::STAGE + Cfg::A_TILE; };

  if (warp < Cfg::PRODUCER_WARP) {
    // ------------------------------------------------------------------ consumers: wgmma + epilogue
    const int wg = warp >> 2;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    float acc[64];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile % p.num_m_blocks;
      const int k_blk = tile / p.num_m_blocks;
      int prev = -1;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t aa = a_addr(stage) + wg * 64 * 128, bb = b_addr(stage);
        wgmma_fence();
#pragma unroll
        for (int s = 0; s < Cfg::RED / 16; ++s) {
          // int4: steps 0..3 reduce the low-nibble plane (A box 0), steps 4..7 the high-nibble plane (A box 1)
          const uint32_t a_s = aa + (s / 4) * Cfg::A_PLANE + (s % 4) * 32;
          const uint32_t b_s = bb + s * 2048;  // 16 reduction rows = two 8-row groups
          wgmma_n128_tb<Cfg::KIND>(acc, wgmma_desc_sw128(a_s), wgmma_desc_sw128_mn(b_s, Cfg::B_ATOM),
                                   (s > 0 || kb > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        wgmma_fence_operands(acc);
        if (prev >= 0 && wg_leader) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == NSTAGES) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      wgmma_fence_operands(acc);
      if (prev >= 0 && wg_leader) mbar_arrive(&empty_bar[prev]);
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
  } else if (warp == Cfg::PRODUCER_WARP) {
    // ------------------------------------------------------------------ TMA producer (gO)
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m_blk = tile % p.num_m_blocks;
        for (int kb = 0; kb < kblocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          mbar_arrive_expect_tx(&full_bar[stage], Cfg::A_TILE);
          uint8_t* dst = smem + stage * Cfg::STAGE;
          if constexpr (Cfg::INT4) {
            tma_load_3d(dst, &tmap_g, &full_bar[stage], kb * 64, 0, m_blk * Cfg::BM);
            tma_load_3d(dst + Cfg::A_PLANE, &tmap_g, &full_bar[stage], kb * 64, 1, m_blk * Cfg::BM);
          } else {
            tma_load_2d(dst, &tmap_g, &full_bar[stage], kb * 64, m_blk * Cfg::BM);
          }
          if (++stage == NSTAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ------------------------------------------------------------------ weight staging
    const int ct = threadIdx.x - Cfg::FIRST_CVT_WARP * 32;
    const int grp = ct / 64;  // staging group == pipeline slot it owns
    const int r = ct % 64;
    const int my_tiles = (num_tiles > static_cast<int>(blockIdx.x))
                             ? (num_tiles - 1 - static_cast<int>(blockIdx.x)) / static_cast<int>(gridDim.x) + 1
                             : 0;
    const int total_it = my_tiles * kblocks;
    const uint32_t bt = b_addr(grp);
    const uint32_t full_addr = smem_u32(full_bar) + grp * 8, empty_addr = smem_u32(empty_bar) + grp * 8;
    const uint32_t sw = static_cast<uint32_t>(r) & 7;
    const uint32_t off_r = (static_cast<uint32_t>(r) >> 3) * 1024 + (static_cast<uint32_t>(r) & 7) * 128;
    int f_it = grp;
    int f_kb = grp % kblocks;
    int f_tile = blockIdx.x + (grp / kblocks) * gridDim.x;
    auto advance = [&]() {
      f_it += NSTAGES;
      f_kb += NSTAGES;
      while (f_kb >= kblocks) { f_kb -= kblocks; f_tile += gridDim.x; }
    };
    uint32_t phase = 0;
    auto publish = [&]() {
      fence_proxy_async_smem();  // generic-proxy stores -> visible to the async proxy (wgmma)
      __syncwarp();
      if (lane == 0) mbar_arrive_u32(full_addr);
      phase ^= 1u;
    };

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
        bool ok;
      };
      auto load_pre = [&](Pre& pr) {
        if (f_it >= total_it) return;
        const int rp = f_kb * 64 + r;
        const int k0 = (f_tile / p.num_m_blocks) * 128;
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
            uint32_t slo, shi, zlo, zhi;
            slo = __ldg(static_cast<const uint16_t*>(p.wscale) + row_lo + g);
            shi = __ldg(static_cast<const uint16_t*>(p.wscale) + row_hi + g);
            if (ZP) {
              zlo = __ldg(static_cast<const uint8_t*>(p.wshift) + row_lo + g);
              zhi = __ldg(static_cast<const uint8_t*>(p.wshift) + row_hi + g);
            } else {
              zlo = __ldg(static_cast<const uint16_t*>(p.wshift) + row_lo + g);
              zhi = __ldg(static_cast<const uint16_t*>(p.wshift) + row_hi + g);
            }
            pr.s[st] = slo | (shi << 16);
            pr.z[st] = zlo | (zhi << 16);
          }
        }
        advance();
      };
      auto process = [&](const Pre& cur) {
        mbar_wait_u32(empty_addr, phase ^ 1u);
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
            const uint32_t atom = bt + (v / 4) * Cfg::B_ATOM + off_r;
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
              st_shared_v4(bt + a * Cfg::B_ATOM + off_r + (c << 4), 0u, 0u, 0u, 0u);
              st_shared_v4(bt + a * Cfg::B_ATOM + off_r + 8 * 1024 + (c << 4), 0u, 0u, 0u, 0u);
            }
        }
        publish();
      };
      Pre pa, pb;
      pa.ok = pb.ok = false;
      load_pre(pa);
      for (int it = grp; it < total_it; it += 2 * NSTAGES) {
        load_pre(pb);
        process(pa);
        if (it + NSTAGES < total_it) {
          load_pre(pa);
          process(pb);
        }
      }
    } else {
      // ---------------- 8-bit weights: thread r converts reduction row n = kb * 64 + r, rnd(scale[n] * W[n, k])
      struct PreB {
        uint4 raw[8];
        uint32_t s2;
      };
      const WT* scale = static_cast<const WT*>(p.wscale);
      auto load_pre = [&](PreB& pr) {
        if (f_it >= total_it) return;
        const int n = f_kb * 64 + r;
        const int k0 = (f_tile / p.num_m_blocks) * 128;
        const bool ok = n < p.N;
        const uint8_t* src = p.w + static_cast<size_t>(ok ? n : 0) * p.K + k0;
#pragma unroll
        for (int v = 0; v < 8; ++v)
          pr.raw[v] = (ok && k0 + v * 16 < p.K) ? __ldg(reinterpret_cast<const uint4*>(src + v * 16)) : make_uint4(0, 0, 0, 0);
        // rows past N: zero bytes times a zero scale -> exact zeros (their gO columns are zero-filled as well)
        const WT sv = ok ? scale[n] : from_float<WT>(0.f);
        pr.s2 = static_cast<uint32_t>(*reinterpret_cast<const uint16_t*>(&sv)) * 0x00010001u;
        advance();
      };
      auto process = [&](const PreB& cur) {
        mbar_wait_u32(empty_addr, phase ^ 1u);
#pragma unroll
        for (int v = 0; v < 8; ++v) {
          uint32_t o[8];
          cvt_bytes4<WT, Cfg::WKIND>(cur.raw[v].x, cur.s2, o[0], o[1]);
          cvt_bytes4<WT, Cfg::WKIND>(cur.raw[v].y, cur.s2, o[2], o[3]);
          cvt_bytes4<WT, Cfg::WKIND>(cur.raw[v].z, cur.s2, o[4], o[5]);
          cvt_bytes4<WT, Cfg::WKIND>(cur.raw[v].w, cur.s2, o[6], o[7]);
          const uint32_t atom = bt + (v / 4) * Cfg::B_ATOM + off_r;
          st_shared_v4(atom + (((2u * (v % 4) + 0u) ^ sw) << 4), o[0], o[1], o[2], o[3]);
          st_shared_v4(atom + (((2u * (v % 4) + 1u) ^ sw) << 4), o[4], o[5], o[6], o[7]);
        }
        publish();
      };
      PreB pa, pb;
      load_pre(pa);
      for (int it = grp; it < total_it; it += 2 * NSTAGES) {
        load_pre(pb);
        process(pa);
        if (it + NSTAGES < total_it) {
          load_pre(pa);
          process(pb);
        }
      }
    }
  }
}

}  // namespace qb
