// The pipeline skeleton of the persistent, warp-specialised wgmma kernels (gemm_tc_kernel, gemm_dgrad_kernel).
//
// One CTA per SM loops over output tiles; a tile's reduction runs through a ring of NSTAGES shared-memory stages, each
// with a `full` and an `empty` mbarrier.  Roles:
//   warps [0, 4*MWG)  consumers      : one warpgroup per 64 rows of the tile issues wgmma on a full stage, keeps one
//                                      stage of MMAs in flight and gives the stage before it back (one arrive on
//                                      `empty` per warpgroup)
//   warp 4*MWG        TMA producer   : waits for an empty stage, arms `full` with the bytes it loads, issues the loads
//   further warps     staging groups : group g (CVT_GROUP_WARPS warps) owns stage slot g and fills every NSTAGES-th
//                                      stage of the CTA's sequence from registers it prefetched; one arrive on `full`
//                                      per warp once its shared-memory stores are visible to the async proxy
// What a stage holds, how it is loaded and converted, and the MMAs and epilogue belong to the kernels; they come in
// here as template parameters and inlined callables.
#pragma once

#include <type_traits>

#include "common.cuh"

namespace qb {

// Warp roles and shared-memory budget from the kernel's tile choices.  TMA_ARRIVALS: arrivals of the TMA producer on
// `full` per stage (0 when the staging warps write every operand); GROUP_WARPS: staging warps per stage slot;
// EPI_BYTES: the consumers' output staging tiles, after the stages (a multiple of 1024 bytes, 0 when there are none);
// GATHER_WARPS: warps after the staging warps that write every stage's A tile from registers (conv_tc.cuh), one arrive
// on `full` each per stage -- they take the place of the TMA producer's arrive.
template <int MWG_, int NSTAGES_, int A_TILE_, int B_TILE_, int GROUP_WARPS_, int TMA_ARRIVALS_, int EPI_BYTES_ = 0,
          int GATHER_WARPS_ = 0>
struct PipeLayout {
  static constexpr int MWG = MWG_;
  static constexpr int NSTAGES = NSTAGES_;
  static constexpr int A_TILE = A_TILE_;
  static constexpr int STAGE = A_TILE_ + B_TILE_;
  static constexpr int CVT_GROUP_WARPS = GROUP_WARPS_;
  static constexpr int NCVT_WARPS = NSTAGES * CVT_GROUP_WARPS;
  static constexpr int PRODUCER_WARP = 4 * MWG;
  static constexpr int FIRST_CVT_WARP = PRODUCER_WARP + 1;
  static constexpr int GATHER_WARPS = GATHER_WARPS_;
  static constexpr int FIRST_GATHER_WARP = FIRST_CVT_WARP + NCVT_WARPS;
  static constexpr int NTHREADS = (FIRST_GATHER_WARP + GATHER_WARPS) * 32;
  static constexpr int FULL_ARRIVALS = TMA_ARRIVALS_ + CVT_GROUP_WARPS + GATHER_WARPS;
  static constexpr int EPI_BYTES = EPI_BYTES_;
  static_assert(EPI_BYTES % 1024 == 0, "output staging tiles keep the 1024-byte alignment of the swizzle");
  // 1024 bytes of alignment slack (the swizzled tiles need 1024-byte aligned bases) + the output staging + the barriers
  static constexpr int SMEM_BYTES = 1024 + NSTAGES * STAGE + EPI_BYTES + 2 * NSTAGES * 8;
  static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");
};

// (stage, phase) of a walk around the ring
template <int NSTAGES>
struct RingPos {
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void advance() {
    if (++stage == NSTAGES) { stage = 0; phase ^= 1u; }
  }
};

// (iteration, k-block, tile) of the CTA's stage sequence that a staging group fills: it = grp, grp + NSTAGES, ...
template <int NSTAGES>
struct StageSeq {
  int it, kb, tile;
  __device__ __forceinline__ StageSeq(int grp, int kblocks)
      : it(grp), kb(grp % kblocks), tile(static_cast<int>(blockIdx.x) + (grp / kblocks) * static_cast<int>(gridDim.x)) {}
  __device__ __forceinline__ void next(int kblocks) {
    it += NSTAGES;
    kb += NSTAGES;
    while (kb >= kblocks) { kb -= kblocks; tile += gridDim.x; }
  }
};

template <class L>
struct WgmmaPipe {
  static constexpr int NSTAGES = L::NSTAGES;
  uint8_t* smem;       // stage 0; stage s at smem + s * STAGE, its A tile first, then its B tile
  uint32_t base;       // shared-memory address of stage 0
  uint32_t epi;        // shared-memory address of the output staging tiles (EPI_BYTES, 1024-byte aligned)
  uint64_t* full_bar;  // [NSTAGES]: the stage's operands have landed
  uint64_t* empty_bar; // [NSTAGES]: every consumer warpgroup is done reading the stage

  // Carves the dynamic shared memory and, from the producer thread, runs `prefetch` (the tensor-map prefetches) and
  // initialises the barriers.  Every thread of the CTA calls it.
  template <class Prefetch>
  __device__ __forceinline__ static WgmmaPipe init(Prefetch&& prefetch) {
    extern __shared__ uint8_t smem_raw[];
    // the swizzled operand tiles need 1024-byte aligned bases (SMEM_BYTES reserves the slack)
    const uint32_t raw_addr = smem_u32(smem_raw);
    WgmmaPipe pipe;
    pipe.smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
    pipe.base = smem_u32(pipe.smem);
    pipe.epi = pipe.base + NSTAGES * L::STAGE;
    pipe.full_bar = reinterpret_cast<uint64_t*>(pipe.smem + NSTAGES * L::STAGE + L::EPI_BYTES);
    pipe.empty_bar = pipe.full_bar + NSTAGES;
    if (threadIdx.x == L::PRODUCER_WARP * 32) {
      prefetch();
      for (int s = 0; s < NSTAGES; ++s) {
        mbar_init(&pipe.full_bar[s], L::FULL_ARRIVALS);
        mbar_init(&pipe.empty_bar[s], L::MWG);  // one arrive per consumer warpgroup
      }
      fence_mbar_init();
    }
    __syncthreads();
    return pipe;
  }

  __device__ __forceinline__ uint32_t a_addr(int s) const { return base + s * L::STAGE; }
  __device__ __forceinline__ uint32_t b_addr(int s) const { return base + s * L::STAGE + L::A_TILE; }

  // Consumers: the k-blocks of one tile.  mma(a, b, accumulate) issues one stage's MMAs, where `a` is this warpgroup's
  // 64 rows of the stage's A tile (128-byte rows) and `b` the stage's B tile; `accumulate` is false for the first stage.
  template <class Acc, int N, class Mma>
  __device__ __forceinline__ void consume_tile(RingPos<NSTAGES>& pos, int kblocks, Acc (&acc)[N], Mma&& mma) const {
    const int wg = static_cast<int>(threadIdx.x >> 5) >> 2;
    const bool wg_leader = (threadIdx.x & 127) == 0;
    int prev = -1;
    for (int kb = 0; kb < kblocks; ++kb) {
      mbar_wait(&full_bar[pos.stage], pos.phase);
      const uint32_t aa = a_addr(pos.stage) + wg * 64 * 128, bb = b_addr(pos.stage);
      wgmma_fence();
      mma(aa, bb, kb > 0);
      wgmma_commit();
      // keep one stage of MMAs in flight; the stage before it has been read and goes back to the producers
      wgmma_wait<1>();
      wgmma_fence_operands(acc);
      if (prev >= 0 && wg_leader) mbar_arrive(&empty_bar[prev]);
      prev = pos.stage;
      pos.advance();
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    if (prev >= 0 && wg_leader) mbar_arrive(&empty_bar[prev]);
  }

  // TMA producer (one thread): every k-block of every tile of this CTA; tile t is output block (t % num_m_blocks,
  // t / num_m_blocks).  load(dst, bar, m_blk, n_blk, kb) issues the loads of one stage into `dst`, completing on `bar`,
  // for `tx_bytes` in all.
  template <class Load>
  __device__ __forceinline__ void produce(int num_tiles, int num_m_blocks, int kblocks, uint32_t tx_bytes,
                                          Load&& load) const {
    RingPos<NSTAGES> pos;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile % num_m_blocks;
      const int n_blk = tile / num_m_blocks;
      for (int kb = 0; kb < kblocks; ++kb) {
        mbar_wait(&empty_bar[pos.stage], pos.phase ^ 1u);
        mbar_arrive_expect_tx(&full_bar[pos.stage], tx_bytes);
        load(smem + pos.stage * L::STAGE, &full_bar[pos.stage], m_blk, n_blk, kb);
        pos.advance();
      }
    }
  }
};

// One thread of a staging group.  The group owns stage slot `grp` and fills stages grp, grp + NSTAGES, ... of the CTA's
// my_tiles x kblocks sequence; the shared code keeps the sequence and the barrier phase, the kernel loads and converts.
template <class L>
struct StagingThread {
  static constexpr int NSTAGES = L::NSTAGES;
  static constexpr int GT = L::CVT_GROUP_WARPS * 32;  // threads per staging group
  int grp, r;       // slot the group owns, thread index within the group
  int kblocks, total_it;
  uint32_t bt;      // the slot's B tile
  uint32_t full_addr, empty_addr;
  uint32_t phase = 0;
  StageSeq<NSTAGES> fetch;  // the next stage to prefetch
  StageSeq<NSTAGES> work;   // the next stage to write

  __device__ __forceinline__ StagingThread(const WgmmaPipe<L>& pipe, int num_tiles, int kblocks_)
      : grp(static_cast<int>(threadIdx.x - L::FIRST_CVT_WARP * 32) / GT),
        r(static_cast<int>(threadIdx.x - L::FIRST_CVT_WARP * 32) % GT), kblocks(kblocks_), fetch(grp, kblocks_),
        work(grp, kblocks_) {
    const int my_tiles = (num_tiles > static_cast<int>(blockIdx.x))
                             ? (num_tiles - 1 - static_cast<int>(blockIdx.x)) / static_cast<int>(gridDim.x) + 1
                             : 0;
    total_it = my_tiles * kblocks;
    bt = pipe.b_addr(grp);
    full_addr = smem_u32(pipe.full_bar) + grp * 8;
    empty_addr = smem_u32(pipe.empty_bar) + grp * 8;
  }

  __device__ __forceinline__ void wait_empty() const { mbar_wait_u32(empty_addr, phase ^ 1u); }
  // every writer: generic-proxy stores -> visible to the async proxy (wgmma); then one arrive per warp
  __device__ __forceinline__ void publish() {
    fence_proxy_async_smem();
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive_u32(full_addr);
    phase ^= 1u;
  }

  // load(pr, seq): read the operands of stage `seq` into registers; past the group's last stage nothing is read
  template <class Pre, class Load>
  __device__ __forceinline__ void prefetch(Pre& pr, Load& load) {
    if (fetch.it >= total_it) return;
    load(pr, static_cast<const StageSeq<NSTAGES>&>(fetch));
    fetch.next(kblocks);
  }

  // process(pr[, seq]): wait_empty(), write the stage from the registers `pr`, publish().  Only a stager that asks for
  // the stage's (k-block, tile) gets `work` kept for it: a stager that does not would pay registers for it.
  template <class Pre, class Process>
  __device__ __forceinline__ void write(const Pre& pr, Process& process) {
    if constexpr (std::is_invocable_v<Process&, const Pre&, const StageSeq<NSTAGES>&>) {
      process(pr, static_cast<const StageSeq<NSTAGES>&>(work));
      work.next(kblocks);
    } else {
      process(pr);
    }
  }

  // The group's stages with ping-pong prefetch buffers (no register copies: copying a register that a load is still
  // filling would stall on the load).  The group's next stage is NSTAGES pipeline stages ahead: ample time to cover L2
  // latency.
  template <class Pre, class Load, class Process>
  __device__ __forceinline__ void run_ping_pong(Load&& load, Process&& process) {
    Pre pa, pb;
    prefetch(pa, load);
    for (int it = grp; it < total_it; it += 2 * NSTAGES) {
      prefetch(pb, load);
      write(pa, process);
      if (it + NSTAGES < total_it) {
        prefetch(pa, load);
        write(pb, process);
      }
    }
  }

  // The same with one stage in registers at a time, for stagers that have no registers for a second buffer.
  template <class Pre, class Load, class Process>
  __device__ __forceinline__ void run_single(Load&& load, Process&& process) {
    for (int it = grp; it < total_it; it += NSTAGES) {
      Pre pa;
      prefetch(pa, load);
      write(pa, process);
    }
  }
};

}  // namespace qb
