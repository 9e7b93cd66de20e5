// Implicit-GEMM 2-D convolution with quantized weights on the wgmma pipeline (Hopper, sm_90a).
//
//   out[b, n, oh, ow] = sum_k im2col(x)[m, k] * W[n, k]       m = (b, oh, ow),  k = c * kh * kw + r * kw + s
//
// A conv weight [Cout, Cin, kh, kw] quantized along axis 0 is, byte for byte, the linear weight [N = Cout, K = Cin*kh*kw]
// (its row-major flattening walks k in the (c, r, s) order above), so the weight operand is staged exactly as for the
// linear (gemm_tc.cuh: stage_weights, int4 or 8-bit with the reference's dequantisation).  Only the A operand and the
// output layout differ.  Roles (wgmma_pipe.cuh):
//   warps [0, 4*MWG)  consumers      : wgmma, then the epilogue straight from the accumulators into the NCHW output
//   warp 4*MWG        (idle)         : initialises the barriers; there is no TMA operand
//   staging warps                    : the weight tile, as in gemm_tc_kernel
//   gather warps      (BM / 32)      : thread t owns row t (one output pixel) of every A tile and writes its 64 k of the
//                                      stage: 64 element loads from the NCHW input -- coalesced across the warp, whose
//                                      32 pixels are mostly consecutive output columns -- then eight 16-byte st.shared
//                                      at the SWIZZLE_128B positions.  Taps in the zero padding and k >= K read 0.
// Developer knock-outs (`make KNOCKOUTS=1` only, GemmParams::dbg; results are wrong while set): 8 = the gather issues
// no loads (it still writes the stage), 256 = the epilogue stores nothing.
// Neither an im2col buffer nor a dequantised weight exists in HBM.  M tiles run over B * Ho * Wo as one dimension: a
// tile may hold the end of one image and the start of the next.
#pragma once

#include "gemm_tc.cuh"

namespace qb {

struct ConvGeom {
  const void* x;  // input [B, C, H, W], NCHW-contiguous, of the 16-bit activation dtype (element alignment only)
  int C, H, W;
  int Ho, Wo;     // output size; M = B * Ho * Wo, the output is [B, N, Ho, Wo] contiguous
  int kh, kw, sh, sw, ph, pw, dh, dw;
};

// The linear's configuration G with its TMA producer replaced by BM / 32 gather warps and no output staging tile.
template <class G>
struct ConvCfg : G {
  static constexpr int GATHER_WARPS = G::BM / 32;
  using Pipe = PipeLayout<G::MWG, G::NSTAGES, G::A_TILE, G::B_TILE, G::BN / 64, 0, 0, GATHER_WARPS>;
  static_assert(G::BSRC == BSrc::INT4 || G::BSRC == BSrc::BYTES, "conv: int4 or weight-only 8-bit weights");
};

// Epilogue of one consumer thread: rows r0 and r0 + 8 of the tile, column pairs 8 j + 2 (lane % 4) of the fragment.
// out = rnd(acc + bias): the bias is added to the fp32 sum and the result rounded once, as the reference's QConv2d
// computes F.conv2d(x, Wd, bias) on the CPU (bit-identical there).  ATen's CUDA path (cuDNN, then a separate bias
// add in the dtype) rounds twice, rnd(rnd(acc) + bias).  Int4 tiles hold the low-nibble out-features
// n_blk * 64 + c in columns [0, 64) and the high-nibble ones N/2 + n_blk * 64 + c - 64 in [64, 128); 8-bit tiles hold
// n_blk * 128 + column.  Stores are 2-byte NCHW stores: the 8 lanes of one column write 8 consecutive pixels.
template <typename OT, bool INT4>
__device__ __forceinline__ void conv_epilogue(const GemmParams& p, const float (&acc)[64], int r0, int n_blk, int lane,
                                              int hw_out) {
  const OT* bias = static_cast<const OT*>(p.bias);
  OT* out = static_cast<OT*>(p.out);
  const int half_n = p.N / 2;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = r0 + 8 * h;
    if (m >= p.M) continue;
    const int b = m / hw_out;
    OT* px = out + static_cast<size_t>(b) * p.N * hw_out + (m - b * hw_out);
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const int col = 8 * j + 2 * (lane & 3);
      int n, n_limit;
      if constexpr (INT4) {
        n = (j < 8) ? n_blk * 64 + col : half_n + n_blk * 64 + col - 64;
        n_limit = (j < 8) ? half_n : p.N;
      } else {
        n = n_blk * 128 + col;
        n_limit = p.N;
      }
      if (n >= n_limit) continue;
      const bool two = n + 1 < n_limit;
      float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
      if (bias != nullptr) {
        f0 = __fadd_rn(f0, to_float<OT>(bias[n]));
        if (two) f1 = __fadd_rn(f1, to_float<OT>(bias[n + 1]));
      }
      if (QB_KO(p.dbg, 256)) continue;  // developer knock-out: no output stores
      px[static_cast<size_t>(n) * hw_out] = from_float<OT>(f0);
      if (two) px[static_cast<size_t>(n + 1) * hw_out] = from_float<OT>(f1);
    }
  }
}

template <class Cfg>
__global__ void __launch_bounds__(Cfg::Pipe::NTHREADS, 1) conv_tc_kernel(const GemmParams p, const ConvGeom c) {
  using L = typename Cfg::Pipe;
  constexpr int BN = Cfg::BN;
  constexpr int BM = Cfg::BM;
  static_assert(BN == 128, "conv: tile width");

  const auto pipe = WgmmaPipe<L>::init([] {});
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.num_m_blocks * p.num_n_blocks;
  const int kblocks = (p.K + 63) / 64;  // 64 16-bit k per stage
  const int hw_out = c.Ho * c.Wo;

  if (warp < L::PRODUCER_WARP) {
    // ------------------------------------------------------------------ consumers: wgmma + NCHW epilogue
    const int wg = warp >> 2;
    float acc[Cfg::NACC];
    RingPos<L::NSTAGES> pos;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m_blk = tile % p.num_m_blocks;
      const int n_blk = tile / p.num_m_blocks;
      pipe.consume_tile(pos, kblocks, acc, [&](uint32_t aa, uint32_t bb, bool accumulate) {
        wgmma_slab<Cfg::KIND, BN>(acc, aa, bb, accumulate);
      });
      conv_epilogue<typename Cfg::WT, Cfg::BSRC == BSrc::INT4>(p, acc, m_blk * BM + wg * 64 + (warp & 3) * 16 + (lane >> 2),
                                                               n_blk, lane, hw_out);
    }
  } else if (warp >= L::FIRST_GATHER_WARP) {
    // ------------------------------------------------------------------ activation gather: row gr of every A tile
    const int gr = static_cast<int>(threadIdx.x) - L::FIRST_GATHER_WARP * 32;
    const uint32_t sw = static_cast<uint32_t>(gr) & 7;
    const uint32_t row_off = (static_cast<uint32_t>(gr) >> 3) * 1024 + sw * 128;
    const uint16_t* x = static_cast<const uint16_t*>(c.x);
    const int khw = c.kh * c.kw;
    const size_t plane = static_cast<size_t>(c.H) * c.W;  // elements of one input channel
    RingPos<L::NSTAGES> pos;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m = (tile % p.num_m_blocks) * BM + gr;
      const bool m_ok = m < p.M;
      int ih0 = 0, iw0 = 0;
      size_t img = 0;  // first element of the pixel's image
      if (m_ok) {
        const int b = m / hw_out, pix = m - b * hw_out;
        const int oh = pix / c.Wo, ow = pix - oh * c.Wo;
        ih0 = oh * c.sh - c.ph;
        iw0 = ow * c.sw - c.pw;
        img = static_cast<size_t>(b) * c.C * plane;
      }
      for (int kb = 0; kb < kblocks; ++kb) {
        const int kbase = kb * 64;
        // tap (ci, r, s) of k = kbase, then stepped along k: s fastest, then r, then the channel
        const int ci = kbase / khw, rs = kbase - ci * khw;
        int r = rs / c.kw, s = rs - (rs / c.kw) * c.kw;
        int ih = ih0 + r * c.dh, iw = iw0 + s * c.dw;
        size_t cofs = img + static_cast<size_t>(ci) * plane;
        uint32_t v[32];
#pragma unroll
        for (int j = 0; j < 64; ++j) {
          uint32_t e = 0;
          if (m_ok && kbase + j < p.K && static_cast<unsigned>(ih) < static_cast<unsigned>(c.H) &&
              static_cast<unsigned>(iw) < static_cast<unsigned>(c.W) && !QB_KO(p.dbg, 8))
            e = __ldg(x + cofs + static_cast<size_t>(ih) * c.W + iw);
          if (j & 1) v[j >> 1] |= e << 16;
          else v[j >> 1] = e;
          if (++s == c.kw) {
            s = 0;
            iw = iw0;
            if (++r == c.kh) {
              r = 0;
              ih = ih0;
              cofs += plane;
            } else {
              ih += c.dh;
            }
          } else {
            iw += c.dw;
          }
        }
        mbar_wait(&pipe.empty_bar[pos.stage], pos.phase ^ 1u);
        const uint32_t dst = pipe.a_addr(pos.stage) + row_off;
#pragma unroll
        for (int ch = 0; ch < 8; ++ch)
          st_shared_v4(dst + ((static_cast<uint32_t>(ch) ^ sw) << 4), v[4 * ch], v[4 * ch + 1], v[4 * ch + 2], v[4 * ch + 3]);
        fence_proxy_async_smem();  // generic-proxy stores -> visible to wgmma
        __syncwarp();
        if (lane == 0) mbar_arrive(&pipe.full_bar[pos.stage]);
        pos.advance();
      }
    }
  } else if (warp > L::PRODUCER_WARP) {
    stage_weights<Cfg>(pipe, p, num_tiles, kblocks);
  }
}

}  // namespace qb
