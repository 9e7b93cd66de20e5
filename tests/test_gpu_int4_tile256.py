"""The swap-AB int4 kernel at its 256-token tile (gemm_tc.cuh: gemm_w4_kernel, T = 256).

A tile is 256 tokens x 64 packed rows; each consumer warpgroup owns 32 packed rows as one m64 fragment and issues one
wgmma.m64n256k16 per k16 step.  The tests run every instantiation at its edges:
- an odd number of 64-row packed blocks, and N / 2 % 64 in {16, 48};
- M one past a 256 boundary, M = 300 and M = 4096;
- fewer tiles than SMs;
- a K tail with groups of 32, zero-points and float shifts, bf16 and fp16, bias, coefficient arrays that start at
  unaligned addresses, and the ordinary-store epilogue.
Every output must be bit-identical to the OVR_TILE_M = 64 route (the 64-token swap kernel, or the weight-staging kernel
where that one runs: same operands, same k order per output element) and pass the float64 oracle bound.
OVR_TILE_M = 256 selects this kernel at any shape.  The fused gather runs it at M = 4096 in
test_gpu_bench_shapes.py::test_fused_gather_emulated_on_one_gpu.
"""
import numpy as np
import pytest
import torch

from helpers import O, bits_to_torch, check_linear, make_qbits_weights, native
from test_gpu_int4_swap import _offset_copy, _overrides, _run

pytestmark = pytest.mark.gpu


# (M, N, K, G)
SHAPES = [
    (3000, 8224, 96, 32),      # ragged M and N / 2, K tail with groups of 32, odd packed-row blocks (65)
    (4097, 6144, 192, 64),     # M one past a 256 boundary (and a 4096 one), even packed-row blocks
    (4096, 14368, 128, 128),   # N / 2 % 64 == 16, 113 packed-row blocks
    (300, 14432, 160, 32),     # M = 300, N / 2 % 64 == 48, K tail with groups of 32
    (257, 33792, 128, 128),    # M one past 256 on the widest grid
    (300, 384, 256, 128),      # 3 packed-row blocks x 2 token blocks: fewer tiles than SMs
    (40, 1048, 64, 64),        # one token block, N % 16 != 0 (ordinary stores), 9 packed-row blocks
]


@pytest.mark.parametrize("tag,zp", [("bf16", False), ("f16", True), ("bf16", True), ("f16", False)])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{m}x{n}x{k}g{g}" for m, n, k, g in SHAPES])
def test_tile256_against_oracle_and_64_token_tile(shape, tag, zp):
    M, N, K, G = shape
    rng = np.random.default_rng(M + N + K)
    _, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=N + K, zeropoint=zp)
    deq_bits = O.dequantize_qbits(packed, 4, scale, shift, tag, N, K, G, shift_is_int=zp)
    x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
    bias_bits = O.from_f32(rng.standard_normal(N, dtype=np.float32), tag) if (M + N) % 3 else None
    x = bits_to_torch(x_bits, tag)
    packed_t = torch.from_numpy(packed).cuda()
    scale_t = _offset_copy(bits_to_torch(scale, tag), 1)
    shift_t = _offset_copy(torch.from_numpy(shift).cuda() if zp else bits_to_torch(shift, tag), 1)
    bias_t = None if bias_bits is None else bits_to_torch(bias_bits, tag)
    staged = _run(x, packed_t, scale_t, shift_t, bias_t, N, K, G, 256, direct=False)
    direct = _run(x, packed_t, scale_t, shift_t, bias_t, N, K, G, 256, direct=True)
    ref64 = _run(x, packed_t, scale_t, shift_t, bias_t, N, K, G, 64, direct=False)
    torch.cuda.synchronize()
    assert torch.equal(staged, direct), (shape, tag, zp)
    assert torch.equal(staged, ref64), (shape, tag, zp)
    check_linear(staged, x_bits, deq_bits, bias_bits, tag, (shape, tag, zp))


def test_tile256_writes_nothing_outside_the_output():
    """The TMA stores of the ragged last token block (a 256-row box) stay inside [M, N]: guard rows before and after the
    output keep their bits."""
    M, N, K, G, tag = 300, 384, 256, 128, "bf16"
    _, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=5)
    x = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    packed_t, scale_t, shift_t = torch.from_numpy(packed).cuda(), bits_to_torch(scale, tag), bits_to_torch(shift, tag)
    n = native()
    lib = n.load()
    buf = torch.full((M + 512, N), 3.0, dtype=torch.bfloat16, device="cuda")
    out = buf[256:256 + M]
    with _overrides(256):
        n.check(lib.qb200_qbits_mm(n.ptr(x), n.ptr(packed_t), n.ptr(scale_t), n.ptr(shift_t), None, n.ptr(out), M, N, K, G,
                                   4, n.DTYPE_CODE[x.dtype], 0, None, 0, n.stream_ptr(x.device)), "qbits_mm")
    ref = _run(x, packed_t, scale_t, shift_t, None, N, K, G, 64, direct=False)
    torch.cuda.synchronize()
    assert bool((buf[:256] == 3.0).all()) and bool((buf[256 + M:] == 3.0).all())
    assert torch.equal(out, ref)
