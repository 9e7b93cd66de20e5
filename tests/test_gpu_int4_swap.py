"""The swap-AB int4 kernel (gemm_tc.cuh: gemm_w4_kernel), which runs the int4 linear once its tiles fill the GPU.

It computes out^T = Wdeq x^T with the dequantised weight as the wgmma register operand.  A tile is T tokens (64 or 128,
test override OVR_TILE_M) x 128 packed rows.  The shapes below take that kernel at both T on a 132-SM H100
(api_qbits.cu: use_swap_kernel), and the tests run every instantiation at its edges against the float64 oracle: M not
a multiple of T, N / 2 not a multiple of 128, a K tail with groups of 32, and scales / shifts that start at any byte
(they are fetched as the aligned 4-byte words that hold them).
"""
import contextlib

import numpy as np
import pytest
import torch

from helpers import O, bits_to_torch, check_linear, make_qbits_weights, native

pytestmark = pytest.mark.gpu
TDT = {"f16": torch.float16, "bf16": torch.bfloat16}


def _overrides(tile_m=None, direct=False):
    n = native()
    stack = contextlib.ExitStack()
    stack.enter_context(n.test_override(n.OVR_INT4_ROUTE, n.ROUTE_INT4_GENERAL))
    if tile_m:
        stack.enter_context(n.test_override(n.OVR_TILE_M, tile_m))
    if direct:
        stack.enter_context(n.test_override(n.OVR_INT4_EPILOGUE, 1))
    return stack


def _offset_copy(t, elems):
    """`t` copied into a buffer `elems` elements past its start: the copy starts at an address that is not 4-byte
    aligned for elems odd."""
    buf = torch.empty(t.numel() + elems, dtype=t.dtype, device="cuda")
    view = buf[elems:].view(t.shape)
    view.copy_(t)
    return view


def _run(x, packed, scale, shift, bias, N, K, G, tile_m, direct):
    n = native()
    lib = n.load()
    out = torch.empty(x.shape[0], N, dtype=x.dtype, device="cuda")
    with _overrides(tile_m, direct):
        n.check(lib.qb200_qbits_mm(n.ptr(x), n.ptr(packed), n.ptr(scale), n.ptr(shift), n.ptr(bias), n.ptr(out),
                                   x.shape[0], N, K, G, 4, n.DTYPE_CODE[x.dtype],
                                   0 if shift.dtype.is_floating_point else 1, None, 0, n.stream_ptr(x.device)),
                "qbits_mm")
        assert lib.qb200_last_kernel_family() == 1
    return out


# (M, N, K, G): ragged M, ragged N / 2 (except 6144), K tails with groups of 32
SHAPES = [(3000, 8224, 96, 32), (1025, 14400, 256, 128), (4097, 6144, 192, 64), (3000, 8224, 160, 32)]


@pytest.mark.parametrize("tile_m", [64, 128])
@pytest.mark.parametrize("tag,zp", [("bf16", False), ("f16", True), ("bf16", True), ("f16", False)])
@pytest.mark.parametrize("shape", SHAPES, ids=[f"{m}x{n}x{k}g{g}" for m, n, k, g in SHAPES])
def test_swap_against_oracle(shape, tag, zp, tile_m):
    M, N, K, G = shape
    rng = np.random.default_rng(M + N + K)
    _, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=N + K, zeropoint=zp)
    deq_bits = O.dequantize_qbits(packed, 4, scale, shift, tag, N, K, G, shift_is_int=zp)
    x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
    bias_bits = O.from_f32(rng.standard_normal(N, dtype=np.float32), tag) if M % 2 else None
    x = bits_to_torch(x_bits, tag)
    packed_t = torch.from_numpy(packed).cuda()
    # scales one element and shifts one element past an aligned start
    scale_t = _offset_copy(bits_to_torch(scale, tag), 1)
    shift_t = _offset_copy(torch.from_numpy(shift).cuda() if zp else bits_to_torch(shift, tag), 1)
    bias_t = None if bias_bits is None else bits_to_torch(bias_bits, tag)
    staged = _run(x, packed_t, scale_t, shift_t, bias_t, N, K, G, tile_m, direct=False)
    direct = _run(x, packed_t, scale_t, shift_t, bias_t, N, K, G, tile_m, direct=True)
    torch.cuda.synchronize()
    assert torch.equal(staged, direct), (shape, tag, zp, tile_m)
    check_linear(staged, x_bits, deq_bits, bias_bits, tag, (shape, tag, zp, tile_m))


@pytest.mark.parametrize("tile_m", [64, 128])
def test_swap_equals_tile_variants_and_unaligned_coefficients(tile_m):
    """The bits do not depend on the token tile, nor on where the coefficient arrays start."""
    M, N, K, G, tag = 4097, 6144, 512, 128, "bf16"
    _, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=3)
    x = torch.randn(M, K, device="cuda").to(TDT[tag])
    packed_t = torch.from_numpy(packed).cuda()
    s, z = bits_to_torch(scale, tag), bits_to_torch(shift, tag)
    ref = _run(x, packed_t, s, z, None, N, K, G, None, direct=False)
    for off in (1, 2, 3):
        out = _run(x, packed_t, _offset_copy(s, off), _offset_copy(z, off), None, N, K, G, tile_m, direct=False)
        torch.cuda.synchronize()
        assert torch.equal(out, ref), (tile_m, off)
