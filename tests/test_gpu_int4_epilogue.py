"""The two epilogues of the int4 wgmma kernel (gemm_tc.cuh: int4_epilogue).

Each consumer warpgroup rounds its 64 x 128 output tile into a swizzled shared-memory tile.  A dense [M, N] output with
N % 16 == 0 is then written with TMA stores through the [M, 2, N/2] plane map; every other output (the fused gather,
N % 16 != 0) and the test override OVR_INT4_EPILOGUE = 1 copy the tile out with ordinary stores.  Both must give the
same bits; the TMA store must write nothing outside the [M, N] output, and must not overwrite a staging tile that a
previous store still reads.
"""
import contextlib

import numpy as np
import pytest
import torch

from helpers import O, bits_to_torch, check_linear, make_qbits_weights, native

pytestmark = pytest.mark.gpu
TDT = {"f16": torch.float16, "bf16": torch.bfloat16}
SENTINEL = 0x5A5A  # bit pattern of the guard bands (a finite value in both 16-bit dtypes)


def _overrides(tile_m=None, direct=False):
    n = native()
    stack = contextlib.ExitStack()
    stack.enter_context(n.test_override(n.OVR_INT4_ROUTE, n.ROUTE_INT4_GENERAL))  # the wgmma kernel at every M
    if tile_m:
        stack.enter_context(n.test_override(n.OVR_TILE_M, tile_m))
    if direct:
        stack.enter_context(n.test_override(n.OVR_INT4_EPILOGUE, 1))
    return stack


def _weights(N, K, G, tag, zp, seed):
    """Device int4 weights: random packed bytes, positive scales, float shifts around 8 * scale or uint8 zero-points."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    dt = TDT[tag]
    packed = torch.randint(0, 256, (N // 2, K), dtype=torch.uint8, device="cuda", generator=gen)
    scale = (torch.rand(N, K // G, device="cuda", generator=gen) * 0.01 + 0.002).to(dt)
    if zp:
        shift = torch.randint(0, 16, (N, K // G), dtype=torch.uint8, device="cuda", generator=gen)
    else:
        shift = (scale.float() * (7 + 2 * torch.rand(N, K // G, device="cuda", generator=gen))).to(dt)
    return packed, scale, shift


def _qbits_mm(x, packed, scale, shift, bias, N, K, G, out):
    """qb200_qbits_mm into the caller's `out` ([M, N] elements, possibly a view into a larger buffer); asserts that the
    wgmma kernel ran."""
    n = native()
    lib = n.load()
    M = x.shape[0]
    n.check(lib.qb200_qbits_mm(n.ptr(x), n.ptr(packed), n.ptr(scale), n.ptr(shift), n.ptr(bias), n.ptr(out), M, N, K, G,
                               4, n.DTYPE_CODE[x.dtype], 0 if shift.dtype.is_floating_point else 1, None, 0,
                               n.stream_ptr(x.device)), "qbits_mm")
    assert lib.qb200_last_kernel_family() == 1
    return out


def _both(x, w, bias, N, K, G, tile_m=None):
    """(TMA-store epilogue, ordinary-store epilogue) outputs of one problem."""
    outs = []
    for direct in (False, True):
        out = torch.empty(x.shape[0], N, dtype=x.dtype, device="cuda")
        with _overrides(tile_m, direct):
            _qbits_mm(x, *w, bias, N, K, G, out)
        outs.append(out)
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("tile_m", [64, 128])
@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("zp", [False, True], ids=["float_shift", "zero_point"])
def test_staged_matches_direct(tile_m, tag, zp):
    """Bit-identical outputs at ragged M (one row past a warpgroup, a tile, two tiles) and N / 2 % 64 in {0, 16, 48}, with
    and without bias."""
    K, G = 256, 128
    for N in (4096, 4128, 4192):
        w = _weights(N, K, G, tag, zp, seed=N + tile_m)
        for M in (17, 65, 127, 129, 300, 4096):
            x = torch.randn(M, K, device="cuda").to(TDT[tag])
            for bias in (None, torch.randn(N, device="cuda").to(TDT[tag])):
                staged, direct = _both(x, w, bias, N, K, G, tile_m)
                assert torch.equal(staged, direct), (tile_m, tag, zp, N, M, bias is not None)


@pytest.mark.parametrize("K,G", [(64, 32), (128, 64)])
@pytest.mark.parametrize("tile_m", [64, 128])
def test_many_tiles_short_reduction(K, G, tile_m):
    """M = 2048 with one or two k-blocks per tile: every warpgroup writes its staging tile again a few microseconds after
    the previous TMA store of it was issued."""
    M, N, tag = 2048, 4192, "bf16"
    w = _weights(N, K, G, tag, False, seed=K)
    x = torch.randn(M, K, device="cuda").to(TDT[tag])
    bias = torch.randn(N, device="cuda").to(TDT[tag])
    staged, direct = _both(x, w, bias, N, K, G, tile_m)
    assert torch.equal(staged, direct), (K, tile_m)


@pytest.mark.parametrize("tile_m", [64, 128])
@pytest.mark.parametrize("M,N", [(129, 4128), (300, 4192), (17, 4096)])
def test_guard_bands_untouched(tile_m, M, N):
    """The output lies inside a larger buffer, 16-byte aligned, between two bands of a sentinel pattern: the TMA store
    writes exactly the [M, N] output and nothing past its last row or before its first."""
    K, G, tag = 128, 64, "bf16"
    band = 128 * N + 8  # a whole 128-row tile past the end; a multiple of 8 elements keeps the 16-byte alignment
    w = _weights(N, K, G, tag, False, seed=M + N)
    x = torch.randn(M, K, device="cuda").to(TDT[tag])
    buf = torch.full((band + M * N + band,), SENTINEL, dtype=torch.int16, device="cuda")
    out = buf[band:band + M * N].view(TDT[tag]).view(M, N)
    assert out.data_ptr() % 16 == 0
    with _overrides(tile_m):
        _qbits_mm(x, *w, None, N, K, G, out)
    ref = torch.empty(M, N, dtype=TDT[tag], device="cuda")
    with _overrides(tile_m, direct=True):
        _qbits_mm(x, *w, None, N, K, G, ref)
    torch.cuda.synchronize()
    assert bool((buf[:band] == SENTINEL).all()), "store before the output"
    assert bool((buf[band + M * N:] == SENTINEL).all()), "store past the output"
    assert torch.equal(out, ref)


@pytest.mark.parametrize("tag,zp", [("bf16", False), ("f16", True)])
def test_staged_against_oracle(tag, zp):
    """The TMA-store epilogue at a ragged shape, with bias, against the float64 oracle (not only against the other
    epilogue)."""
    M, N, K, G = 129, 4128, 256, 128
    rng = np.random.default_rng(5)
    _, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=7, zeropoint=zp)
    deq_bits = O.dequantize_qbits(packed, 4, scale, shift, tag, N, K, G, shift_is_int=zp)
    x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
    bias_bits = O.from_f32(rng.standard_normal(N, dtype=np.float32), tag)
    shift_t = torch.from_numpy(shift).cuda() if zp else bits_to_torch(shift, tag)
    out = torch.empty(M, N, dtype=TDT[tag], device="cuda")
    with _overrides():
        _qbits_mm(bits_to_torch(x_bits, tag), torch.from_numpy(packed).cuda(), bits_to_torch(scale, tag), shift_t,
                  bits_to_torch(bias_bits, tag), N, K, G, out)
    torch.cuda.synchronize()
    check_linear(out, x_bits, deq_bits, bias_bits, tag, (tag, zp))


@pytest.mark.parametrize("tag", ["bf16", "f16"])
def test_n_not_multiple_of_16_uses_ordinary_stores(tag):
    """N % 16 != 0 (plane rows not 16-byte aligned) takes the ordinary-store epilogue: against the oracle, with bias, and
    equal to the forced ordinary-store run."""
    M, N, K, G = 130, 4104, 128, 64
    rng = np.random.default_rng(9)
    _, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=11)
    deq_bits = O.dequantize_qbits(packed, 4, scale, shift, tag, N, K, G)
    x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
    bias_bits = O.from_f32(rng.standard_normal(N, dtype=np.float32), tag)
    w = (torch.from_numpy(packed).cuda(), bits_to_torch(scale, tag), bits_to_torch(shift, tag))
    auto, direct = _both(bits_to_torch(x_bits, tag), w, bits_to_torch(bias_bits, tag), N, K, G)
    assert torch.equal(auto, direct)
    check_linear(auto, x_bits, deq_bits, bias_bits, tag, tag)
