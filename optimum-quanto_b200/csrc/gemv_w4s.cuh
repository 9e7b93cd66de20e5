// Batch-1..8 decode ("gemv") fused packed-int4 linear: a TMA-fed shared-memory ring, whole-K ownership per CTA.
//
// The register-streaming kernel in gemv_w4.cuh keeps at most 4 x 16 B per thread in flight and splits K across CTAs
// (stream-K), so a 30 MB weight matrix was read at ~1.3 TB/s with a 5.6 us cross-CTA fix-up at the end.  Here:
//   * every CTA owns a contiguous range of PACKED rows (= out-feature pairs n, n + N/2) over the whole K, so there is
//     no split-K, no workspace, no tickets and the result is deterministic by construction;
//   * one elected thread streams those rows with cp.async.bulk (TMA, 1-D) into a ring that holds ~190 KB per SM --
//     132 SMs x 190 KB is the whole matrix in flight at launch, HBM never waits for an instruction to be issued;
//   * 16 compute warps read the ring with conflict-free LDS.128 (rows padded by 64 B), dequantise in registers with the
//     reference's rounding order (tensor/qbits.py:34-45) and accumulate with mma.sync.m16n8k16: MMA rows 0-7 are the
//     low nibbles of 8 packed rows, rows 8-15 their high nibbles, the 8 MMA columns are the (<= 8) tokens;
//   * the activations sit in shared memory (M x K), a 17th warp is the TMA producer, an 18th reduces the 16 per-warp
//     partial tiles of a row group in a fixed order and writes the outputs.
// Stage = (group of <= 8 packed rows) x (KC k-bytes); a warp handles a contiguous run of 64-byte slabs of each stage.
// The scales / shifts of a row group (4 contiguous runs: scale and shift of the low- and high-nibble features) travel
// through their own small TMA ring one or more groups ahead: read with LDG at first use they cost a DRAM round trip per
// row group (measured: 28 us per launch against 12 us for the weight stream alone).
#pragma once

#include "gather.cuh"
#include "gemv_w4.cuh"

namespace qb {

struct GemvSParams {
  const uint8_t* wq;   // [N/2, K] packed bytes
  const void* scale;   // [N * K / group]
  const void* shift;   // same shape (weight dtype, or uint8 zero-points)
  const void* bias;    // [N] or nullptr
  const void* x;       // [M, K]
  void* out;           // [M, ld] (this rank's buffer; ld = N, col0 = 0 for an ordinary call)
  GatherInfo g;        // fused all-gather of a column-parallel linear (gather.cuh); g.n_out == 1: ordinary call
  int ld, col0;
  int M, N, K;
  int group, group_log2;
  int KC;              // k-bytes per stage (divides K, multiple of 64)
  int nkc;             // K / KC
  int nstages;         // ring depth
  int stage_bytes;     // 8 * (KC + 64)
  int x_stride;        // bytes per token row in shared memory (K * 2 + 16: conflict-free LDS.128 across tokens)
  int cdepth;          // coefficient ring depth (row groups)
  int coef_arr;        // bytes of one coefficient array of a slot: 8 rows x (K / group) x 2
  int dbg;
  int pmode;           // producer issue mode (see the producer warp)
  long long* trace;    // developer timeline: CTA < 4, [cta][2][32] clock64 stamps (row 0 compute warp 0, row 1 producer)
};

constexpr int kGemvSDefaultProducer = 1;  // measured: one lane per packed row (8 x 4 KB copies in flight per issue)
constexpr int kGemvSComputeWarps = 16;
constexpr int kGemvSThreads = (kGemvSComputeWarps + 2) * 32;
constexpr int kGemvSRedBytes = 2 * kGemvSComputeWarps * 128 * 4;

__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void bulk_load_1d(uint32_t smem_dst, const void* src, uint32_t bytes, uint32_t bar,
                                             uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_dst),
      "l"(src), "r"(bytes), "r"(bar), "l"(policy)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx_u32(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ uint2 ld_shared_v2(uint32_t addr) {
  uint2 v;
  asm volatile("ld.shared.v2.b32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr) : "memory");
  return v;
}

// KO: developer knock-outs (compile-time, so the shipped loop carries no extra branches):
//   1 no dequant arithmetic, 2 no tensor-core instruction, 3 no nibble extraction either (dequant + extraction off)
//   CR: scales / shifts come through the coefficient ring (else LDG at first use: rows of scales not 16-byte multiples)
template <typename WT, bool ZP, bool CR, int KO = 0>
__global__ void __launch_bounds__(kGemvSThreads, 1) gemv_w4s_kernel(const GemvSParams p) {
  using D = Dq<WT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 127) & ~uintptr_t(127));
  const uint32_t ring = smem_u32(smem);
  uint8_t* coef = smem + static_cast<size_t>(p.nstages) * p.stage_bytes;                         // [cdepth][4][coef_arr]
  float* red = reinterpret_cast<float*>(coef + static_cast<size_t>(p.cdepth) * 4 * p.coef_arr);  // [2][16][128]
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(red) + kGemvSRedBytes);
  // bars: full[nstages], empty[nstages], red_full[2], red_empty[2], coef_full[cdepth], coef_empty[cdepth]
  const uint32_t full0 = smem_u32(bars), empty0 = full0 + p.nstages * 8;
  const uint32_t red_full0 = empty0 + p.nstages * 8, red_empty0 = red_full0 + 16;
  const uint32_t cfull0 = red_empty0 + 16, cempty0 = cfull0 + p.cdepth * 8;
  const uint32_t coef_addr = smem_u32(coef);
  uint8_t* xs = reinterpret_cast<uint8_t*>(bars + 2 * p.nstages + 4 + 2 * p.cdepth);
  const uint32_t xs_addr = smem_u32(xs);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int half_n = p.N / 2;
  const int r_begin = static_cast<int>(static_cast<int64_t>(blockIdx.x) * half_n / gridDim.x);
  const int r_end = static_cast<int>(static_cast<int64_t>(blockIdx.x + 1) * half_n / gridDim.x);
  const int ngroups = (r_end - r_begin + 7) / 8;
  const int row_pitch = p.KC + 64;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nstages; ++s) {
      mbar_init(&bars[s], 1);
      mbar_init(&bars[p.nstages + s], kGemvSComputeWarps);
    }
    for (int b = 0; b < 2; ++b) {
      mbar_init(&bars[2 * p.nstages + b], kGemvSComputeWarps);
      mbar_init(&bars[2 * p.nstages + 2 + b], 1);
    }
    for (int c = 0; c < p.cdepth; ++c) {
      mbar_init(&bars[2 * p.nstages + 4 + c], 1);
      mbar_init(&bars[2 * p.nstages + 4 + p.cdepth + c], kGemvSComputeWarps);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();  // the next kernel may start its weight stream on every SM this grid frees

  if (warp == kGemvSComputeWarps) {
    // ------------------------------------------------------------------ TMA producer (whole warp)
    // One thread arms the stage's barrier; the copies of a stage are then issued by several lanes at once.  A single
    // thread sustains one cp.async.bulk per ~380 cycles (tools/tma_probe.cu), i.e. ~11 B/cycle/SM with 4 KB copies
    // against the 22 B/cycle/SM share of HBM -- with one issuing thread the ring feed, not HBM, bounded this kernel
    // (12 us for the stream alone, round 1).  pmode 1: one lane per packed row; 2: 32 lanes = (row, k quarter);
    // 0: the single-thread producer (kept for comparison, tools/gemv_probe.py).
    const uint64_t pol = l2_policy_evict_first();
    const int pmode = p.pmode;
    int s = 0, pc = 0;
    uint32_t phase = 0, pcph = 0;
    int tn = 0;
    auto stamp = [&]() {
      if (p.trace != nullptr && blockIdx.x < 4 && lane == 0 && tn < 32) p.trace[(blockIdx.x * 2 + 1) * 32 + tn++] = clock64();
    };
    stamp();
    for (int gi = 0; gi < ngroups; ++gi) {
      const int r0 = r_begin + gi * 8;
      const int rows = min(8, r_end - r0);
      if (CR) {  // scales / shifts of this row group: 4 contiguous runs of rows x (K / group) entries
        const int c = pc;
        const int gpr = p.K / p.group;
        const uint32_t sbytes = static_cast<uint32_t>(rows) * gpr * 2, zbytes = ZP ? sbytes / 2 : sbytes;
        if (lane == 0) {
          mbar_wait_u32(cempty0 + c * 8, pcph ^ 1u);
          mbar_arrive_expect_tx_u32(cfull0 + c * 8, 2 * sbytes + 2 * zbytes);
        }
        __syncwarp();
        const size_t lo = static_cast<size_t>(r0) * gpr, hi = lo + static_cast<size_t>(p.N / 2) * gpr;
        const uint32_t dst = coef_addr + c * 4 * p.coef_arr;
        const uint8_t* sc = static_cast<const uint8_t*>(p.scale);
        const uint8_t* zs = static_cast<const uint8_t*>(p.shift);
        for (int a = (pmode == 0 ? 0 : lane); a < 4; a += (pmode == 0 ? 1 : 32)) {
          if (pmode == 0 && lane != 0) break;
          const uint8_t* src = (a == 0) ? sc + lo * 2 : (a == 1) ? sc + hi * 2 : (a == 2) ? zs + lo * (ZP ? 1 : 2) : zs + hi * (ZP ? 1 : 2);
          bulk_load_1d(dst + a * p.coef_arr, src, a < 2 ? sbytes : zbytes, cfull0 + c * 8, pol);
        }
        if (++pc == p.cdepth) { pc = 0; pcph ^= 1u; }
      }
      for (int kc = 0; kc < p.nkc; ++kc) {
        if (lane == 0) {
          mbar_wait_u32(empty0 + s * 8, phase ^ 1u);
          mbar_arrive_expect_tx_u32(full0 + s * 8, static_cast<uint32_t>(rows) * p.KC);
        }
        __syncwarp();
        const uint8_t* src = p.wq + static_cast<size_t>(r0) * p.K + static_cast<size_t>(kc) * p.KC;
        const uint32_t dst = ring + s * p.stage_bytes;
        if (pmode == 0) {
          if (lane == 0)
            for (int r = 0; r < rows; ++r)
              bulk_load_1d(dst + r * row_pitch, src + static_cast<size_t>(r) * p.K, p.KC, full0 + s * 8, pol);
        } else if (pmode == 1) {
          if (lane < rows)
            bulk_load_1d(dst + lane * row_pitch, src + static_cast<size_t>(lane) * p.K, p.KC, full0 + s * 8, pol);
        } else {
          const int r = lane & 7, qd = lane >> 3;
          const uint32_t part = static_cast<uint32_t>(p.KC) >> 2;  // KC % 64 == 0: 16-byte multiples
          if (r < rows)
            bulk_load_1d(dst + r * row_pitch + qd * part, src + static_cast<size_t>(r) * p.K + qd * part, part,
                         full0 + s * 8, pol);
        }
        stamp();
        if (++s == p.nstages) { s = 0; phase ^= 1u; }
      }
    }
    return;
  }

  if (warp == kGemvSComputeWarps + 1) {
    // ------------------------------------------------------------------ reducer: 16 partial tiles -> outputs
    for (int gi = 0; gi < ngroups; ++gi) {
      const int b = gi & 1;
      const uint32_t ph = (gi >> 1) & 1u;
      const int r0 = r_begin + gi * 8;
      const int rows = min(8, r_end - r0);
      mbar_wait_u32(red_full0 + b * 8, ph);
      const float* rb = red + b * (kGemvSComputeWarps * 128);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int o = lane + 32 * q;      // o = tile row * 8 + token
        const int trow = o >> 3, tok = o & 7;
        float sum = 0.f;
#pragma unroll
        for (int w = 0; w < kGemvSComputeWarps; ++w) sum += rb[w * 128 + o];
        if (tok < p.M && (trow & 7) < rows) {
          const int n = (trow < 8) ? (r0 + trow) : (half_n + r0 + trow - 8);
          WT r = from_float<WT>(sum);
          if (p.bias != nullptr)
            r = from_float<WT>(__fadd_rn(to_float<WT>(r), to_float<WT>(static_cast<const WT*>(p.bias)[n])));
          const size_t o_idx = static_cast<size_t>(tok) * p.ld + p.col0 + n;
          static_cast<WT*>(p.out)[o_idx] = r;
          for (int q = 1; q < p.g.n_out; ++q) static_cast<WT*>(p.g.out_peer[q])[o_idx] = r;  // peers, over NVLink
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive_u32(red_empty0 + b * 8);
    }
    __syncwarp();  // this warp made every output store of the CTA
    if (lane == 0) gather_signal_end(p.g);
    return;
  }

  // -------------------------------------------------------------------- compute warps
  // activations -> shared memory (the producer is already streaming weights)
  {
    const int ct = threadIdx.x;  // 0 .. 511
    pdl_wait();  // the activations (and the gather flags) are the previous kernel's output; the weight stream is running
    if (p.g.n_out > 1 && p.g.wait_start) {  // the activation is the gathered output of the previous linear
      if (ct == 0) gather_wait_start(p.g);
      asm volatile("bar.sync 1, %0;" ::"n"(kGemvSComputeWarps * 32) : "memory");
    }
    const int vec_per_row = p.K / 8;  // 16-byte vectors per token row
    for (int i = ct; i < p.M * vec_per_row; i += kGemvSComputeWarps * 32) {
      const int m = i / vec_per_row, v = i - m * vec_per_row;
      // plain (coherent) load: with a gathered input these bytes were written by peers during the previous kernel
      const uint4 val = *reinterpret_cast<const uint4*>(static_cast<const uint8_t*>(p.x) +
                                                        (static_cast<size_t>(m) * p.K + v * 8) * 2);
      *reinterpret_cast<uint4*>(xs + static_cast<size_t>(m) * p.x_stride + v * 16) = val;
    }
    asm volatile("bar.sync 1, %0;" ::"n"(kGemvSComputeWarps * 32) : "memory");
  }

  const int g = lane >> 2;  // packed row inside the group (MMA rows g and g + 8), and the token column of B
  const int t = lane & 3;   // owns bytes [16t, 16t + 16) of every 64-byte slab
  const int gpr = p.K / p.group;  // groups per out-feature row
  const bool tok_ok = g < p.M;
  const uint32_t x_lane = xs_addr + g * p.x_stride;
  const int nslabs = p.KC / 64;
  const int spw = (nslabs + kGemvSComputeWarps - 1) / kGemvSComputeWarps;  // slabs per warp and stage (contiguous run)
  const int sl_begin = min(warp * spw, nslabs), sl_end = min(sl_begin + spw, nslabs);

  int s = 0;
  uint32_t phase = 0;
  int tn = 0;
  auto stamp = [&]() {
    if (p.trace != nullptr && blockIdx.x < 4 && threadIdx.x == 0 && tn < 32) p.trace[(blockIdx.x * 2) * 32 + tn++] = clock64();
  };
  stamp();
  constexpr bool coef_ring = CR;
  int cs = 0;                           // coefficient ring slot / phase of the current row group
  uint32_t cphase = 0;
  // one slab's worth of operands, loaded one slab ahead of its use (weights, the lane's 16 activations, raw coefficients)
  struct Pre {
    uint4 w, xa, xc;
    uint16_t s_lo, s_hi, z_lo, z_hi;
    int qg;
  };
  for (int gi = 0; gi < ngroups; ++gi) {
    const int r0 = r_begin + gi * 8;
    const int rows = min(8, r_end - r0);
    const int gr = (g < rows) ? g : 0;  // rows beyond the group: stale ring bytes, masked at the output
    // two accumulators: consecutive k-steps alternate, so the MMAs of a slab are not one dependent chain
    float acc0[4] = {0.f, 0.f, 0.f, 0.f}, acc1[4] = {0.f, 0.f, 0.f, 0.f};
    const size_t q_lo = static_cast<size_t>(r0 + gr) * gpr, q_hi = q_lo + static_cast<size_t>(half_n) * gpr;
    const uint32_t c_lane = coef_addr + cs * 4 * p.coef_arr + gr * gpr * 2;  // this lane's row in the scale arrays
    const uint32_t z_lane = coef_addr + cs * 4 * p.coef_arr + 2 * p.coef_arr + gr * gpr * (ZP ? 1 : 2);
    if (coef_ring) mbar_wait_u32(cfull0 + cs * 8, cphase);
    for (int kc = 0; kc < p.nkc; ++kc) {
      const int kbase = kc * p.KC + t * 16;
      mbar_wait_u32(full0 + s * 8, phase);
      stamp();
      const uint32_t lane_base = ring + s * p.stage_bytes + g * row_pitch + t * 16;
      auto load_pre = [&](Pre& pr, int sl) {
        const int kk = kbase + sl * 64;  // first k of this lane's 16 bytes
        pr.w = ld_shared_v4(lane_base + sl * 64);
        pr.xa = make_uint4(0u, 0u, 0u, 0u);
        pr.xc = make_uint4(0u, 0u, 0u, 0u);
        if (tok_ok) {  // the lane's 16 activations (k = kk .. kk+15) of token g: 32 contiguous bytes
          pr.xa = ld_shared_v4(x_lane + kk * 2);
          pr.xc = ld_shared_v4(x_lane + kk * 2 + 16);
        }
        const int qg = kk >> p.group_log2;  // group sizes are powers of two on this path
        pr.qg = qg;
        if constexpr (!coef_ring) {
          pr.s_lo = __ldg(static_cast<const uint16_t*>(p.scale) + q_lo + qg);
          pr.s_hi = __ldg(static_cast<const uint16_t*>(p.scale) + q_hi + qg);
          if (ZP) {
            pr.z_lo = __ldg(static_cast<const uint8_t*>(p.shift) + q_lo + qg);
            pr.z_hi = __ldg(static_cast<const uint8_t*>(p.shift) + q_hi + qg);
          } else {
            pr.z_lo = __ldg(static_cast<const uint16_t*>(p.shift) + q_lo + qg);
            pr.z_hi = __ldg(static_cast<const uint16_t*>(p.shift) + q_hi + qg);
          }
        } else {
          asm volatile("ld.shared.u16 %0, [%1];" : "=h"(pr.s_lo) : "r"(c_lane + qg * 2));
          asm volatile("ld.shared.u16 %0, [%1];" : "=h"(pr.s_hi) : "r"(c_lane + p.coef_arr + qg * 2));
          if (ZP) {
            asm volatile("ld.shared.u8 %0, [%1];" : "=h"(pr.z_lo) : "r"(z_lane + qg));
            asm volatile("ld.shared.u8 %0, [%1];" : "=h"(pr.z_hi) : "r"(z_lane + p.coef_arr + qg));
          } else {
            asm volatile("ld.shared.u16 %0, [%1];" : "=h"(pr.z_lo) : "r"(z_lane + qg * 2));
            asm volatile("ld.shared.u16 %0, [%1];" : "=h"(pr.z_hi) : "r"(z_lane + p.coef_arr + qg * 2));
          }
        }
      };
      typename D::Coef c_lo, c_hi;
      int cur_qg = -1;
      auto consume = [&](const Pre& pr) {
        if (pr.qg != cur_qg) {  // (scale, shift) of the lane's two out-features changed
          cur_qg = pr.qg;
          c_lo = D::make_raw(*reinterpret_cast<const WT*>(&pr.s_lo), pr.z_lo, ZP);
          c_hi = D::make_raw(*reinterpret_cast<const WT*>(&pr.s_hi), pr.z_hi, ZP);
        }
        const uint32_t w4[4] = {pr.w.x, pr.w.y, pr.w.z, pr.w.w};
        const uint32_t xb[8] = {pr.xa.x, pr.xa.y, pr.xa.z, pr.xa.w, pr.xc.x, pr.xc.y, pr.xc.z, pr.xc.w};
#pragma unroll
        for (int st = 0; st < 4; ++st) {  // k-step: bytes 4st .. 4st+3 = k  kk + 4st .. +3
          uint32_t a[4];
          if constexpr (KO == 3) {
            a[0] = w4[st]; a[1] = w4[st] ^ *reinterpret_cast<const uint32_t*>(&c_lo.s); a[2] = w4[st] + 1u; a[3] = w4[st] ^ *reinterpret_cast<const uint32_t*>(&c_hi.s);
          } else {
            const uint32_t l = w4[st] & 0x0F0F0F0Fu, h = (w4[st] >> 4) & 0x0F0F0F0Fu;
            if constexpr (KO == 1) {
              a[0] = __byte_perm(l, D::MAGIC_BYTES, 0x4140) ^ *reinterpret_cast<const uint32_t*>(&c_lo.s); a[1] = __byte_perm(h, D::MAGIC_BYTES, 0x4140);
              a[2] = __byte_perm(l, D::MAGIC_BYTES, 0x4342) ^ *reinterpret_cast<const uint32_t*>(&c_hi.s); a[3] = __byte_perm(h, D::MAGIC_BYTES, 0x4342);
            } else {
              a[0] = D::cvt(__byte_perm(l, D::MAGIC_BYTES, 0x4140), c_lo, ZP);  // row g   (low nibble),  k slots 2t, 2t+1
              a[1] = D::cvt(__byte_perm(h, D::MAGIC_BYTES, 0x4140), c_hi, ZP);  // row g+8 (high nibble)
              a[2] = D::cvt(__byte_perm(l, D::MAGIC_BYTES, 0x4342), c_lo, ZP);  // row g,   k slots 2t+8, 2t+9
              a[3] = D::cvt(__byte_perm(h, D::MAGIC_BYTES, 0x4342), c_hi, ZP);
            }
          }
          if constexpr (KO == 2) {
            acc0[st] += __uint_as_float(a[0] ^ a[1] ^ a[2] ^ a[3] ^ xb[2 * st] ^ xb[2 * st + 1]);
          } else {
            if (st & 1) mma_m16n8k16<WT>(acc1, a, xb[2 * st], xb[2 * st + 1]);
            else mma_m16n8k16<WT>(acc0, a, xb[2 * st], xb[2 * st + 1]);
          }
        }
      };
      if (sl_begin < sl_end && !QB_KO(p.dbg, 8)) {  // developer switch 8: stream only
        // ping-pong operand buffers, one slab ahead (no register copies of in-flight loads)
        Pre pa, pb;
        load_pre(pa, sl_begin);
        for (int sl = sl_begin; sl < sl_end; sl += 2) {
          if (sl + 1 < sl_end) load_pre(pb, sl + 1);
          consume(pa);
          if (sl + 1 < sl_end) {
            if (sl + 2 < sl_end) load_pre(pa, sl + 2);
            consume(pb);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive_u32(empty0 + s * 8);
      if (++s == p.nstages) { s = 0; phase ^= 1u; }
    }
    __syncwarp();
    if (coef_ring) {
      if (lane == 0) mbar_arrive_u32(cempty0 + cs * 8);
      if (++cs == p.cdepth) { cs = 0; cphase ^= 1u; }
    }
    // ---- this warp's partial 16 x 8 tile -> reducer
    const int b = gi & 1;
    mbar_wait_u32(red_empty0 + b * 8, ((gi >> 1) & 1u) ^ 1u);
    float* rp = red + (b * kGemvSComputeWarps + warp) * 128;
    *reinterpret_cast<float2*>(rp + g * 8 + 2 * t) = make_float2(acc0[0] + acc1[0], acc0[1] + acc1[1]);        // row g
    *reinterpret_cast<float2*>(rp + (g + 8) * 8 + 2 * t) = make_float2(acc0[2] + acc1[2], acc0[3] + acc1[3]);  // row g+8
    __syncwarp();
    if (lane == 0) mbar_arrive_u32(red_full0 + b * 8);
    stamp();
  }
}

}  // namespace qb
