"""GPU parity tests through the C-ABI (include/quanto_b200.h) against the oracle and the golden fixtures."""
import os

import numpy as np
import pytest
import torch

from helpers import (O, bits_to_torch, cabi_dequantize_qbits, cabi_qbits_mm, cabi_qbytes_mm, cabi_quantize_symmetric,
                     cabi_unpack, make_qbits_weights, torch_to_bits, torch_to_f32)
from helpers import check_linear as _check_linear

pytestmark = pytest.mark.gpu


def _load(golden_dir, name):
    return np.load(os.path.join(golden_dir, name))


# ------------------------------------------------------------------------------------------- unpack
def test_unpack_golden(golden_dir):
    z = _load(golden_dir, "unpack.npz")
    for i in range(int(z["n_unpack"])):
        out = cabi_unpack(torch.from_numpy(z[f"c{i}_in"]).cuda(), int(z[f"c{i}_bits"]))
        assert np.array_equal(out.cpu().numpy(), z[f"c{i}_out"]), i


@pytest.mark.parametrize("bits", [2, 4])
@pytest.mark.parametrize("shape", [(1,), (17,), (4099,), (229376, 128), (1000, 24)])
def test_unpack_random(bits, shape):
    g = torch.Generator().manual_seed(1)
    packed = torch.randint(0, 256, shape, dtype=torch.uint8, generator=g)
    out = cabi_unpack(packed.cuda(), bits)
    assert np.array_equal(out.cpu().numpy(), O.unpack(packed.numpy(), bits))


def test_unpack_errors():
    from quanto_b200 import _native as n
    with pytest.raises(ValueError):
        cabi_unpack(torch.zeros(16, dtype=torch.uint8, device="cuda"), 3)
    assert n.load().qb200_unpack(None, None, 0, 4, None) == 0  # empty input is fine


# ------------------------------------------------------------------------------ quantize_symmetric
def test_quantize_symmetric_golden(golden_dir):
    z = _load(golden_dir, "quantize_symmetric.npz")
    for i in range(int(z["n"])):
        p = f"c{i}_"
        in_tag, out_tag = str(z[p + "in_tag"]), str(z[p + "out_tag"])
        axis = int(z[p + "axis"])
        axis = None if axis == -2 else axis
        base = bits_to_torch(z[p + "base"], in_tag)
        scale = bits_to_torch(z[p + "scale"], in_tag)
        out_dtype = {"int8": torch.int8, "e4m3fn": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}[out_tag]
        out = cabi_quantize_symmetric(base, out_dtype, axis, scale)
        assert np.array_equal(torch_to_bits(out).view(np.uint8), z[p + "out"].view(np.uint8)), (i, in_tag, out_tag, axis)


@pytest.mark.parametrize("in_tag", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("out_tag", ["int8", "e4m3fn", "e5m2"])
@pytest.mark.parametrize("axis", [None, 0, -1])
def test_quantize_symmetric_large(in_tag, out_tag, axis):
    rng = np.random.default_rng(3)
    shape = (1024, 2048)
    base = O.round_to(rng.standard_normal(shape, dtype=np.float32) * 2, in_tag)
    if axis is None:
        scale = O.round_to(np.array(np.abs(base).max() / 120, np.float32), in_tag)
    elif axis == 0:
        scale = O.round_to(np.abs(base).max(axis=1, keepdims=True) / 127, in_tag)
    else:
        scale = O.round_to(np.abs(base).max(axis=0, keepdims=True) / 127, in_tag)
    ref = O.quantize_symmetric(base, in_tag, out_tag, scale)
    out_dtype = {"int8": torch.int8, "e4m3fn": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}[out_tag]
    out = cabi_quantize_symmetric(bits_to_torch(O.from_f32(base, in_tag), in_tag), out_dtype, axis,
                                  bits_to_torch(O.from_f32(scale, in_tag), in_tag))
    assert np.array_equal(torch_to_bits(out).view(np.uint8), ref.view(np.uint8))


def test_quantize_symmetric_bf16_all_values():
    """Every finite bf16 value against 48 scales: pins the reciprocal-multiply path of the bf16 kernel bit for bit."""
    bits = np.arange(65536, dtype=np.uint16)
    vals = O.bf16_bits_to_f32(bits)
    bits = bits[np.isfinite(vals)]
    bits = np.resize(bits, (255, 256))  # 65280 finite values, padded by wrap-around to a vectorisable shape
    base = O.bf16_bits_to_f32(bits)
    rng = np.random.default_rng(5)
    scales = np.concatenate([O.round_to(np.exp(rng.uniform(-12, 6, 40)).astype(np.float32), "bf16"),
                             np.array([1.0, 0.5, 3.0, 0.0078125, 1.1754944e-38, 3.0e38, 7.0, 0.33203125], np.float32)])
    for sc in scales:
        sc = O.round_to(np.array(sc, np.float32), "bf16")
        for out_tag, out_dtype in (("int8", torch.int8), ("e4m3fn", torch.float8_e4m3fn)):
            ref = O.quantize_symmetric(base, "bf16", out_tag, sc)
            out = cabi_quantize_symmetric(bits_to_torch(bits, "bf16"), out_dtype, None, bits_to_torch(O.from_f32(sc, "bf16"), "bf16"))
            got = torch_to_bits(out).view(np.uint8)
            assert np.array_equal(got, ref.view(np.uint8)), (float(sc), out_tag, int(np.sum(got != ref.view(np.uint8))))


# ------------------------------------------------------------------------------ dequantize / qbits_mm
def test_dequantize_qbits_golden(golden_dir):
    z = _load(golden_dir, "qbits.npz")
    for i in range(int(z["n"])):
        p = f"c{i}_"
        tag = str(z[p + "tag"])
        N, K, G, M = (int(v) for v in z[p + "shape"])
        zp = bool(int(z[p + "zeropoint"]))
        packed = torch.from_numpy(z[p + "packed"]).cuda()
        scale = bits_to_torch(z[p + "scale"], tag).reshape(-1)
        shift = torch.from_numpy(z[p + "shift"]).cuda().reshape(-1) if zp else bits_to_torch(z[p + "shift"], tag).reshape(-1)
        deq = cabi_dequantize_qbits(packed, scale, shift, N, K, G, int(z[p + "bits"]))
        assert np.array_equal(torch_to_bits(deq), z[p + "deq"]), (i, tag)


def test_qbits_mm_golden(golden_dir):
    z = _load(golden_dir, "qbits.npz")
    ran = 0
    for i in range(int(z["n"])):
        p = f"c{i}_"
        tag = str(z[p + "tag"])
        N, K, G, M = (int(v) for v in z[p + "shape"])
        if tag == "f32" or int(z[p + "bits"]) != 4:
            continue
        zp = bool(int(z[p + "zeropoint"]))
        packed = torch.from_numpy(z[p + "packed"]).cuda()
        scale = bits_to_torch(z[p + "scale"], tag).reshape(-1)
        shift = torch.from_numpy(z[p + "shift"]).cuda().reshape(-1) if zp else bits_to_torch(z[p + "shift"], tag).reshape(-1)
        x = bits_to_torch(z[p + "x"], tag)
        bias = bits_to_torch(z[p + "bias"], tag) if (p + "bias") in z.files else None
        y = cabi_qbits_mm(x, packed, scale, shift, bias, N, K, G)
        torch.cuda.synchronize()
        same = _check_linear(y, z[p + "x"], z[p + "deq"], z[p + "bias"] if bias is not None else None, tag, f"golden{i}")
        # against the reference's own output: identical except where fp32 summation order flips a rounding
        yref = O.to_f32(z[p + "y"], tag).astype(np.float64)
        rel = np.linalg.norm(torch_to_f32(y) - yref) / np.linalg.norm(yref)
        assert rel < 1e-3 and same > 0.97, (i, rel, same)
        ran += 1
    assert ran >= 6


@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("M,N,K,G", [(1, 256, 128, 128), (7, 512, 1024, 128), (128, 256, 256, 64), (129, 768, 512, 128),
                                     (300, 1280, 1024, 128), (512, 4096, 4096, 128), (64, 96, 160, 32)])
@pytest.mark.parametrize("zeropoint", [False, True])
def test_qbits_mm_shapes(tag, M, N, K, G, zeropoint):
    if zeropoint and (M, N) not in ((7, 512), (300, 1280)):
        pytest.skip("zeropoint variant covered on two shapes")
    q, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=M + N, zeropoint=zeropoint)
    rng = np.random.default_rng(M * 7 + K)
    x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
    bias_bits = O.from_f32(rng.standard_normal(N, dtype=np.float32), tag) if (M % 2 == 1) else None
    deq_bits = O.dequantize_qbits(packed, 4, scale, shift, tag, N, K, G, shift_is_int=zeropoint)
    shift_t = torch.from_numpy(shift).cuda() if zeropoint else bits_to_torch(shift, tag)
    y = cabi_qbits_mm(bits_to_torch(x_bits, tag), torch.from_numpy(packed).cuda(), bits_to_torch(scale, tag), shift_t,
                      None if bias_bits is None else bits_to_torch(bias_bits, tag), N, K, G)
    torch.cuda.synchronize()
    # the kernel's dequantisation itself is checked bit-exactly through the standalone dequantize entry point
    deq_gpu = cabi_dequantize_qbits(torch.from_numpy(packed).cuda(), bits_to_torch(scale, tag), shift_t, N, K, G, 4)
    assert np.array_equal(torch_to_bits(deq_gpu), deq_bits)
    _check_linear(y, x_bits, deq_bits, bias_bits, tag, (tag, M, N, K, G))


@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("M,N,K,G", [(1, 14336, 4096, 128), (5, 4096, 4096, 128), (16, 1024, 4096, 128),
                                     (32, 4096, 14336, 128), (33, 1536, 1024, 64), (100, 2048, 1024, 128),
                                     (128, 640, 512, 32), (3, 130, 256, 128)])
def test_qbits_mm_decode_streamk(tag, M, N, K, G):
    """Small-M stream-K kernel: every segment / fix-up pattern (1 segment per block .. many), twice (ticket recycle)."""
    if tag == "f16" and N > 4096:
        pytest.skip("large shapes once (bf16)")
    zeropoint = (M == 5)
    q, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=N + K, zeropoint=zeropoint)
    rng = np.random.default_rng(M + 3 * K)
    x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
    bias_bits = O.from_f32(rng.standard_normal(N, dtype=np.float32), tag) if (M % 2 == 1) else None
    deq_bits = O.dequantize_qbits(packed, 4, scale, shift, tag, N, K, G, shift_is_int=zeropoint)
    shift_t = torch.from_numpy(shift).cuda() if zeropoint else bits_to_torch(shift, tag)
    args = (bits_to_torch(x_bits, tag), torch.from_numpy(packed).cuda(), bits_to_torch(scale, tag), shift_t,
            None if bias_bits is None else bits_to_torch(bias_bits, tag), N, K, G)
    y1 = cabi_qbits_mm(*args)
    y2 = cabi_qbits_mm(*args)
    torch.cuda.synchronize()
    assert torch.equal(y1, y2)  # deterministic split-K reduction, tickets recycled correctly
    _check_linear(y1, x_bits, deq_bits, bias_bits, tag, ("decode", tag, M, N, K, G))
    # the general kernel (no workspace) computes the same operands: results agree up to fp32 summation order
    y3 = cabi_qbits_mm(*args, use_workspace=False)
    torch.cuda.synchronize()
    _check_linear(y3, x_bits, deq_bits, bias_bits, tag, ("general", tag, M, N, K, G))


@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("M,N,K,G", [(1, 4096, 4096, 128), (2, 4096, 14336, 128), (8, 1024, 4096, 32),
                                     (4, 2048, 11008, 128), (3, 130, 256, 64), (6, 298, 192, 64), (8, 14336, 4096, 128),
                                     (1, 2, 64, 32)])
def test_qbits_mm_gemv_ring(tag, M, N, K, G):
    """M <= 8 TMA-ring gemv (gemv_w4s.cuh): ragged row ranges per CTA, multi-chunk K, group 32/64/128, zero-points,
    and agreement with the stream-K kernel it replaces (same operands, fp32 summation order differs)."""
    if tag == "f16" and N * K > 4096 * 4096:
        pytest.skip("large shapes once (bf16)")
    from helpers import native
    zeropoint = (M % 4 == 2)
    q, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=N + K + M, zeropoint=zeropoint)
    rng = np.random.default_rng(M + 5 * K)
    x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
    bias_bits = O.from_f32(rng.standard_normal(N, dtype=np.float32), tag) if (M % 2 == 1) else None
    deq_bits = O.dequantize_qbits(packed, 4, scale, shift, tag, N, K, G, shift_is_int=zeropoint)
    shift_t = torch.from_numpy(shift).cuda() if zeropoint else bits_to_torch(shift, tag)
    args = (bits_to_torch(x_bits, tag), torch.from_numpy(packed).cuda(), bits_to_torch(scale, tag), shift_t,
            None if bias_bits is None else bits_to_torch(bias_bits, tag), N, K, G)
    n = native()
    lib = n.load()
    # forced: the automatic route sends the Llama-sized shapes here to the second-generation kernel instead
    with n.test_override(n.OVR_INT4_ROUTE, n.ROUTE_INT4_RING):
        y1 = cabi_qbits_mm(*args)
        fam = lib.qb200_last_kernel_family()
        y2 = cabi_qbits_mm(*args, use_workspace=False)  # the ring kernel needs no workspace
        torch.cuda.synchronize()
    assert fam == 3
    assert torch.equal(y1, y2)
    _check_linear(y1, x_bits, deq_bits, bias_bits, tag, ("gemv_ring", tag, M, N, K, G))
    y0 = cabi_qbits_mm(*args)  # the dispatcher's own choice passes the same bound
    torch.cuda.synchronize()
    _check_linear(y0, x_bits, deq_bits, bias_bits, tag, ("auto", tag, M, N, K, G))
    if K % 128 == 0:  # the stream-K warp-MMA kernel this one replaced for M <= 8 (still the 8 < M <= 32 candidate)
        with n.test_override(n.OVR_INT4_ROUTE, n.ROUTE_INT4_GEMV):
            y3 = cabi_qbits_mm(*args)
            torch.cuda.synchronize()
        _check_linear(y3, x_bits, deq_bits, bias_bits, tag, ("streamk", tag, M, N, K, G))


@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("M,N,K,G", [(1, 4096, 4096, 128), (2, 4096, 14336, 128), (8, 1024, 4096, 64), (5, 2048, 2048, 128),
                                     (3, 144, 1024, 64), (7, 304, 3072, 64), (8, 14336, 4096, 128), (1, 16, 2048, 128),
                                     (9, 14336, 4096, 128), (16, 4096, 4096, 128), (12, 1024, 4096, 64), (16, 2064, 2048, 128),
                                     (8, 4096, 14336, 128), (4, 2048, 14336, 128), (13, 1024, 4096, 64)])
def test_qbits_mm_gemv_ring2(tag, M, N, K, G):
    """M <= 16 second-generation TMA-ring gemv (gemv_w4r.cuh): whole 8-row groups per CTA, every (slabs per warp, group
    size, token groups) instantiation, one and several passes over K (activations too large for shared memory), zero-points,
    bias, bulk-store output; bit-identical to the first generation wherever both cut K the same way."""
    if tag == "f16" and N * K > 4096 * 4096:
        pytest.skip("large shapes once (bf16)")
    from helpers import native
    n = native()
    zeropoint = (M % 4 == 2)
    q, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=N + K + M, zeropoint=zeropoint)
    rng = np.random.default_rng(M + 5 * K)
    x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
    bias_bits = O.from_f32(rng.standard_normal(N, dtype=np.float32), tag) if (M % 2 == 1) else None
    deq_bits = O.dequantize_qbits(packed, 4, scale, shift, tag, N, K, G, shift_is_int=zeropoint)
    shift_t = torch.from_numpy(shift).cuda() if zeropoint else bits_to_torch(shift, tag)
    args = (bits_to_torch(x_bits, tag), torch.from_numpy(packed).cuda(), bits_to_torch(scale, tag), shift_t,
            None if bias_bits is None else bits_to_torch(bias_bits, tag), N, K, G)
    lib = n.load()
    with n.test_override(n.OVR_INT4_ROUTE, n.ROUTE_INT4_RING2):
        y1 = cabi_qbits_mm(*args)
        fam = lib.qb200_last_kernel_family()
        y2 = cabi_qbits_mm(*args, use_workspace=False)  # no workspace
        torch.cuda.synchronize()
    assert fam == 3
    assert torch.equal(y1, y2)
    _check_linear(y1, x_bits, deq_bits, bias_bits, tag, ("gemv_ring2", tag, M, N, K, G))
    if M <= 2 and K % 2048 == 0:  # the opt-in two-CTAs-per-SM shape (stages of 2048 k): same bound
        with n.test_override(n.OVR_GEMV_SHAPE, 2), n.test_override(n.OVR_INT4_ROUTE, n.ROUTE_INT4_RING2):
            yl = cabi_qbits_mm(*args)
            torch.cuda.synchronize()
        _check_linear(yl, x_bits, deq_bits, bias_bits, tag, ("gemv_ring2_lite", tag, M, N, K, G))
    y0 = cabi_qbits_mm(*args)  # the dispatcher's own choice passes the same bound
    torch.cuda.synchronize()
    _check_linear(y0, x_bits, deq_bits, bias_bits, tag, ("auto", tag, M, N, K, G))
    if M <= 8 and K in (2048, 4096, 8192, 14336) and (M * (K * 2 + 16)) <= 72 * 1024:  # one pass over K in both kernels
        with n.test_override(n.OVR_INT4_ROUTE, n.ROUTE_INT4_RING):
            y3 = cabi_qbits_mm(*args)
            torch.cuda.synchronize()
        assert torch.equal(y1, y3), "first- and second-generation ring kernels cut K identically here"


@pytest.mark.parametrize("tag", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("bits", [4, 2])
@pytest.mark.parametrize("M,N,K,G", [(4, 8, 40, 40), (33, 51, 96, 32), (70, 130, 200, 8), (5, 64, 256, 128), (129, 48, 50, 50)])
def test_qbits_mm_cuda_core_kernel(tag, bits, M, N, K, G):
    """Shapes / types the tensor-core kernels do not take (2-bit weights, odd N, K % 16 != 0, exotic group sizes, fp32,
    per-axis quantisation = one group per row) run on the library's own CUDA-core kernel: same operands, same bound.
    Reference: tests/tensor/ops/test_linear_dispatch.py:27 (qint2 / qint4), tensor/qbits.py:27-49."""
    if bits == 4 and tag != "f32" and (M, N, K, G) == (5, 64, 256, 128):
        pytest.skip("this one is a tensor-core shape")
    rng = np.random.default_rng(M + N + K + bits)
    rows = N * K // G
    qv = rng.integers(0, 1 << bits, size=(rows, G), dtype=np.uint8)
    packed = O.pack_weights(qv, bits)
    scale = O.from_f32(rng.random(rows, dtype=np.float32) * 0.01 + 0.002, tag)
    zeropoint = (M % 2 == 0)
    shift = rng.integers(0, 1 << bits, size=rows, dtype=np.uint8) if zeropoint else O.from_f32(
        O.to_f32(scale, tag) * (1.0 + rng.random(rows, dtype=np.float32)), tag)
    x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
    bias_bits = O.from_f32(rng.standard_normal(N, dtype=np.float32), tag) if N % 2 else None
    deq_bits = O.dequantize_qbits(packed, bits, scale, shift, tag, N, K, G, shift_is_int=zeropoint)
    shift_t = torch.from_numpy(shift).cuda() if zeropoint else bits_to_torch(shift, tag)
    y = cabi_qbits_mm(bits_to_torch(x_bits, tag), torch.from_numpy(packed).cuda(), bits_to_torch(scale, tag), shift_t,
                      None if bias_bits is None else bits_to_torch(bias_bits, tag), N, K, G, bits=bits)
    torch.cuda.synchronize()
    from helpers import native
    assert native().load().qb200_last_kernel_family() == 2
    _check_linear(y, x_bits, deq_bits, bias_bits, tag, ("cuda-core", tag, bits, M, N, K, G))


def test_qbits_mm_errors():
    x = torch.zeros(4, 40, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(ValueError):  # the group must divide K
        cabi_qbits_mm(x, torch.zeros(8 * 40 // 2, dtype=torch.uint8, device="cuda"),
                      torch.ones(8, dtype=torch.bfloat16, device="cuda"), torch.ones(8, dtype=torch.bfloat16, device="cuda"),
                      None, 8, 40, 32)
    with pytest.raises(ValueError):  # the op validates dtypes instead of reinterpreting bits (ADVICE r1)
        torch.ops.quanto.qbits_mm(x, torch.zeros(4, 40, dtype=torch.uint8, device="cuda"),
                                  torch.ones(8, 1, dtype=torch.float16, device="cuda"),
                                  torch.ones(8, 1, dtype=torch.float16, device="cuda"), None, 8, 40)


# --------------------------------------------------------------------------------------- qbytes_mm
def _decode(arr, kind, tag):
    if kind == "int8":
        return arr.astype(np.float32)
    if kind == "same":
        return O.to_f32(arr, tag)
    return O.fp8_bits_to_f32(arr, kind)


def test_qbytes_mm_golden(golden_dir):
    z = _load(golden_dir, "qbytes_mm.npz")
    for i in range(int(z["n"])):
        p = f"c{i}_"
        akind, wkind, tag = str(z[p + "akind"]), str(z[p + "wkind"]), str(z[p + "tag"])
        A = bits_to_torch(z[p + "A"], tag if akind == "same" else akind)
        W = bits_to_torch(z[p + "W"], wkind)
        scales_bits = z[p + "scales"]
        scales = bits_to_torch(scales_bits, tag)
        y, family = cabi_qbytes_mm(A, W, scales.reshape(-1))
        torch.cuda.synchronize()
        s32 = O.to_f32(scales_bits, tag)
        if akind == "int8" and wkind == "int8":
            assert np.array_equal(torch_to_bits(y), z[p + "y"]), (i, tag, family)  # bit exact vs the reference
            continue
        a = _decode(z[p + "A"], akind, tag)
        w = _decode(z[p + "W"], wkind, tag)
        yg = torch_to_f32(y).astype(np.float64)
        if family == 1 and akind in ("e4m3fn", "e5m2"):
            # native fp8 tensor-core path: exact products, scale applied in fp32 after the accumulation
            y64, _ = O.qbytes_mm_fp8_native(z[p + "A"], akind, z[p + "W"], wkind, s32, tag)
            bound = 0.51 * O.ulp(y64, tag) + O.accumulate_allowance(a, w) * np.abs(s32).reshape(1, -1)
            assert np.all(np.abs(yg - y64) <= bound), (i, "native", float(np.max(np.abs(yg - y64) / bound)))
            yref = O.to_f32(z[p + "y"], tag).astype(np.float64)
            rel = np.linalg.norm(yg - yref) / np.linalg.norm(yref)
            # the reference rounds scales*W to the output dtype first (qbytes_mm.py:31-33): documented gap
            assert rel < (2.5e-3 if tag == "bf16" else 6e-4), (i, rel)
            continue
        y64, _ = O.qbytes_mm(a, w, s32, tag)
        ap, wp = O.qbytes_mm_operands(a, w, s32, tag)
        bound = 0.51 * O.ulp(y64, tag) + O.accumulate_allowance(ap, wp)
        assert np.all(np.abs(yg - y64) <= bound), (i, akind, wkind, tag, float(np.max(np.abs(yg - y64) / bound)))


@pytest.mark.parametrize("tag", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("M,N,K", [(17, 48, 64), (256, 1024, 1024), (130, 300, 528), (512, 2048, 4096), (33, 50, 50)])
def test_qbytes_mm_int8_exact(tag, M, N, K):
    rng = np.random.default_rng(M + N + K)
    A = rng.integers(-127, 128, size=(M, K), dtype=np.int8)
    W = rng.integers(-128, 128, size=(N, K), dtype=np.int8)
    s = O.round_to(rng.random(N, dtype=np.float32) / 1e3 + 1e-5, tag)
    bias = O.round_to(rng.standard_normal(N, dtype=np.float32), tag) if M % 2 else None
    y, family = cabi_qbytes_mm(torch.from_numpy(A).cuda(), torch.from_numpy(W).cuda(),
                               bits_to_torch(O.from_f32(s, tag), tag),
                               None if bias is None else bits_to_torch(O.from_f32(bias, tag), tag))
    torch.cuda.synchronize()
    assert family == (1 if K % 16 == 0 else 2)
    ref = O.to_f32(O.qbytes_int_mm(A, W, s, tag), tag)
    if bias is not None:
        ref = O.round_to(ref + bias, tag)
    assert np.array_equal(torch_to_bits(y), O.from_f32(ref, tag)), (tag, M, N, K, family)


@pytest.mark.parametrize("tag", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("M,N,K", [(512, 2048, 4096), (1024, 1024, 512), (384, 4096, 256)])
def test_qbytes_mm_int8_fused_bias_large(tag, M, N, K):
    """Bias fused into the epilogue of the wgmma kernels: acc*scale rounded, then + bias rounded, exactly
    the two roundings of the reference's `qbytes_mm(...) + bias` (tensor/weights/qbytes.py:68-82)."""
    rng = np.random.default_rng(M * 3 + N + K)
    A = rng.integers(-127, 128, size=(M, K), dtype=np.int8)
    W = rng.integers(-128, 128, size=(N, K), dtype=np.int8)
    s = O.round_to(rng.random(N, dtype=np.float32) / 1e3 + 1e-5, tag)
    bias = O.round_to(rng.standard_normal(N, dtype=np.float32), tag)
    y, family = cabi_qbytes_mm(torch.from_numpy(A).cuda(), torch.from_numpy(W).cuda(),
                               bits_to_torch(O.from_f32(s, tag), tag), bits_to_torch(O.from_f32(bias, tag), tag))
    assert family == 1
    ref = O.round_to(O.to_f32(O.qbytes_int_mm(A, W, s, tag), tag) + bias, tag)
    assert np.array_equal(torch_to_bits(y), O.from_f32(ref, tag)), (tag, M, N, K)
    # the op the 8-bit QLinear calls when it has a bias
    y2 = torch.ops.quanto.qbytes_linear(torch.from_numpy(A).cuda(), torch.from_numpy(W).cuda(),
                                        bits_to_torch(O.from_f32(s, tag), tag).reshape(-1, 1),
                                        bits_to_torch(O.from_f32(bias, tag), tag))
    assert torch.equal(y2, y)


@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("wkind", ["int8", "e4m3fn", "e5m2"])
@pytest.mark.parametrize("M,N,K", [(7, 300, 128), (128, 512, 1024), (300, 640, 2048), (1000, 1024, 512)])
def test_qbytes_mm_weight_only_tensor_path(tag, wkind, M, N, K):
    """fp16/bf16 activations x int8/fp8 weights on wgmma: operands rnd(scale*W) are bit-identical to the reference's
    python path (library/qbytes_mm.py:25-33); only the fp32 summation order may differ."""
    rng = np.random.default_rng(M + N + K)
    a = O.round_to(rng.standard_normal((M, K), dtype=np.float32), tag)
    if wkind == "int8":
        w_store = rng.integers(-128, 128, size=(N, K), dtype=np.int8)
        w = w_store.astype(np.float32)
    else:
        w_store = O.f32_to_fp8_bits(np.clip(rng.standard_normal((N, K), dtype=np.float32) * 3, -200, 200), wkind)
        w = O.fp8_bits_to_f32(w_store, wkind)
    s = O.round_to(rng.random(N, dtype=np.float32) / 1e2 + 1e-4, tag)
    bias = O.round_to(rng.standard_normal(N, dtype=np.float32), tag) if M % 2 else None
    y, family = cabi_qbytes_mm(bits_to_torch(O.from_f32(a, tag), tag), bits_to_torch(w_store, wkind),
                               bits_to_torch(O.from_f32(s, tag), tag),
                               None if bias is None else bits_to_torch(O.from_f32(bias, tag), tag))
    torch.cuda.synchronize()
    assert family == 1
    ap, wp = O.qbytes_mm_operands(a, w, s, tag)
    y64, _, tol = O.linear_from_dequantized(ap, wp, bias, tag)
    bound = 1.02 * tol + O.accumulate_allowance(ap, wp)
    err = np.abs(torch_to_f32(y).astype(np.float64) - y64)
    assert np.all(err <= bound), (tag, wkind, M, N, K, float(np.max(err / bound)))


@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("akind,wkind", [("e4m3fn", "e4m3fn"), ("e5m2", "e4m3fn"), ("e4m3fn", "e5m2")])
def test_qbytes_mm_fp8_native(tag, akind, wkind):
    M, N, K = 200, 384, 512
    rng = np.random.default_rng(11)
    a_bits = O.f32_to_fp8_bits(np.clip(rng.standard_normal((M, K), dtype=np.float32), -3, 3), akind)
    w_bits = O.f32_to_fp8_bits(np.clip(rng.standard_normal((N, K), dtype=np.float32) * 2, -6, 6), wkind)
    s = O.round_to(rng.random(N, dtype=np.float32) / 1e2 + 1e-4, tag)
    y, family = cabi_qbytes_mm(bits_to_torch(a_bits, akind), bits_to_torch(w_bits, wkind),
                               bits_to_torch(O.from_f32(s, tag), tag))
    torch.cuda.synchronize()
    assert family == 1
    y64, _ = O.qbytes_mm_fp8_native(a_bits, akind, w_bits, wkind, s, tag)
    a, w = O.fp8_bits_to_f32(a_bits, akind), O.fp8_bits_to_f32(w_bits, wkind)
    bound = 0.51 * O.ulp(y64, tag) + O.accumulate_allowance(a, w) * s.reshape(1, -1)
    yg = torch_to_f32(y).astype(np.float64)
    assert np.all(np.abs(yg - y64) <= bound), float(np.max(np.abs(yg - y64) / bound))
