// Shared between the translation units of the fused packed-int4 linear (api_qbits.cu: dispatcher + wgmma kernel,
// api_qbits_small.cu: gemv kernels).
#pragma once

#include "gather.cuh"
#include "host_common.cuh"

namespace qb {

struct QbitsArgs {
  const void* a;          // [M, K] activations
  const uint8_t* packed;  // canonical packed weights
  const void* scale;
  const void* shift;
  const void* bias;
  void* out;              // this rank's [M, ld] output (== g.out_peer[0])
  int64_t m, n, k;        // n = out-features computed by this call (the local shard of a column-parallel linear)
  int64_t ld, col0;       // row pitch of the output buffers, first column written (ordinary call: ld = n, col0 = 0)
  int group, group_log2, bits;
  int dtype, shift_is_int;
  void* workspace;
  int64_t workspace_bytes;
  GatherInfo g;           // g.n_out == 1: ordinary call
  cudaStream_t stream;
};

int64_t qbits_small_workspace_bytes(int64_t m, int64_t n, int64_t k);
int qbits_ring_plan(int64_t m, int64_t n, int64_t k, int group, int zp, int grid, int* out);
int qbits_small_dispatch(const QbitsArgs& q, bool* handled);

}  // namespace qb
