"""GPU tests through the reference-facing surface: torch.ops.quanto.*, QTensor dispatch, QLinear (vs golden outputs)."""
import os

import numpy as np
import pytest
import torch

import quanto_b200 as q
from helpers import O, bits_to_torch, torch_to_bits, torch_to_f32

pytestmark = pytest.mark.gpu
TDT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}


def tt(arr, dtype):
    if dtype in (torch.float16, torch.bfloat16):
        return torch.from_numpy(arr.view(np.int16).copy()).view(dtype)
    return torch.from_numpy(arr.copy())


def test_unpack_op_and_packed_tensor_roundtrip():
    # reference tests/library/test_unpack.py:22-30 and tests/tensor/test_packed_tensor.py:24-35
    for bits in (2, 4):
        for shape in ((12,), (32, 32), (10, 8), (12, 8)):
            u = torch.randint(0, 2**bits, shape, dtype=torch.uint8)
            p = q.PackedTensor.pack(u.cuda(), bits)
            assert p.device.type == "cuda" and torch.equal(p.unpack().cpu(), u)
            assert torch.equal(torch.ops.quanto.unpack(p._data, bits)[: shape[0]].cpu(), u)
            moved = p.cpu().cuda()
            assert isinstance(moved, q.PackedTensor) and torch.equal(moved.unpack().cpu(), u)


def test_quantize_symmetric_op_validation_and_values():
    base = torch.randn(32, 64, device="cuda", dtype=torch.float16)
    with pytest.raises(ValueError):
        torch.ops.quanto.quantize_symmetric(base, dtype=torch.int8, axis=None, scale=torch.ones(2, device="cuda").half())
    with pytest.raises(ValueError):  # 1-D tensors cannot be quantized per-axis
        torch.ops.quanto.quantize_symmetric(base[0], dtype=torch.int8, axis=0, scale=torch.ones(64, device="cuda").half())
    scale = (base.abs().amax(dim=1, keepdim=True) / 127)
    out = torch.ops.quanto.quantize_symmetric(base, dtype=torch.int8, axis=0, scale=scale)
    ref = O.quantize_symmetric(torch_to_f32(base), "f16", "int8", torch_to_f32(scale))
    assert np.array_equal(out.cpu().numpy(), ref)
    # integer-valued tensors survive exactly (reference tests/library/test_quantize.py:105-119)
    ints = torch.randint(-127, 127, (16, 32)).to(torch.float32).cuda()
    assert torch.equal(torch.ops.quanto.quantize_symmetric(ints, dtype=torch.int8, axis=None,
                                                           scale=torch.tensor(1.0, device="cuda")).float(), ints)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("wq", [q.qint4, q.qint2])
def test_qbits_tensor_dequantize_and_linear_dispatch(dtype, wq):
    torch.manual_seed(0)
    N, K, M = 256, 512, 24
    w = (torch.randn(N, K) * 0.05).to(dtype).cuda()
    scale, shift = q.MaxOptimizer()(w, qtype=wq, axis=0, group_size=128)
    qw = q.quantize_weight(w, qtype=wq, axis=0, scale=scale, shift=shift, group_size=128)
    assert isinstance(qw, q.WeightQBitsTensor) and qw.device.type == "cuda"
    tag = "bf16" if dtype == torch.bfloat16 else "f16"
    deq = qw.dequantize()
    ref = O.dequantize_qbits(qw._data._data.cpu().numpy(), wq.bits, torch_to_bits(qw._scale), torch_to_bits(qw._shift),
                             tag, N, K, 128)
    assert np.array_equal(torch_to_bits(deq), ref)
    x = torch.randn(2, M, K).to(dtype).cuda()
    bias = torch.randn(N).to(dtype).cuda()
    y = torch.nn.functional.linear(x, qw, bias)
    assert y.shape == (2, M, N) and y.dtype == dtype
    y64, _, tol = O.linear_from_dequantized(torch_to_f32(x).reshape(-1, K), O.to_f32(ref, tag), torch_to_f32(bias), tag)
    err = np.abs(torch_to_f32(y).reshape(-1, N).astype(np.float64) - y64)
    bound = 1.02 * tol + O.accumulate_allowance(torch_to_f32(x).reshape(-1, K), O.to_f32(ref, tag))
    assert np.all(err <= bound), float(np.max(err / bound))
    # serialization identity on device
    assert torch.equal(qw.cpu().cuda(), qw)


def test_qlinear_matches_reference_outputs(golden_dir):
    """QLinear outputs of the real reference (CPU, python path) vs our CUDA path on the same state dict and input."""
    z = np.load(os.path.join(golden_dir, "qlinear.npz"))
    for i in range(int(z["n"])):
        p = f"c{i}_"
        tag = str(z[p + "tag"])
        dtype = TDT[tag]
        N, K, M, G = (int(v) for v in z[p + "shape"])
        wq = q.qtypes[str(z[p + "wq"])]
        aq = None if str(z[p + "aq"]) == "none" else q.qtypes[str(z[p + "aq"])]
        lin = torch.nn.Linear(K, N, bias=True).to(dtype)
        ql = q.QLinear.from_module(lin, weights=wq, activations=aq)
        sd = {"bias": tt(z[p + "bias"], dtype), "input_scale": tt(z[p + "input_scale"], dtype).reshape(()),
              "output_scale": tt(z[p + "output_scale"], dtype).reshape(())}
        for key in z.files:
            if key.startswith(p + "sd_"):
                name = key[len(p) + 3:]
                arr = z[key]
                if name.endswith("_data") and wq.bits == 8 and wq.is_floating_point:
                    sd[name] = torch.from_numpy(arr.copy()).view(wq.dtype)
                elif name.endswith("_data") or arr.dtype == np.uint8:
                    sd[name] = torch.from_numpy(arr.copy())
                else:
                    sd[name] = tt(arr, dtype)
        ql.load_state_dict(sd)
        ql = ql.cuda()
        x = tt(z[p + "x"], dtype).cuda()
        with torch.no_grad():
            y = ql(x)
        torch.cuda.synchronize()
        if aq is None:
            yref = O.to_f32(z[p + "y"], tag).astype(np.float64)
            yg = torch_to_f32(y).astype(np.float64)
            rel = np.linalg.norm(yg - yref) / np.linalg.norm(yref)
            same = float(np.mean(torch_to_bits(y) == z[p + "y"]))
            # bf16 x int8 on the reference CPU goes through torch._weight_int8pack_mm (scale after accumulate)
            lim = 4e-3 if (wq.bits == 8 and tag == "bf16") else 1e-3
            assert rel < lim, (i, str(z[p + "wq"]), tag, rel, same)
        else:
            assert isinstance(y, q.ActivationQBytesTensor)
            ref_data = z[p + "y_data"].view(np.uint8).astype(np.int16)
            got = torch_to_bits(y._data).view(np.uint8).astype(np.int16)
            if aq.is_floating_point:
                mismatch = np.mean(got != ref_data)
                assert mismatch < 0.05, (i, mismatch)
            else:
                d = np.abs(got.astype(np.int8).astype(np.int16) - ref_data.astype(np.int8).astype(np.int16))
                assert d.max() <= 1 and np.mean(d != 0) < 0.05, (i, int(d.max()), float(np.mean(d != 0)))


def test_qlinear_int8_activations_bit_exact_chain():
    """int8 activations x int8 weights: quantize_symmetric + qbytes_mm + quantize_output all bit-exact vs the oracle."""
    torch.manual_seed(3)
    K, N, M = 256, 128, 64
    dtype, tag = torch.bfloat16, "bf16"
    lin = torch.nn.Linear(K, N, bias=False).to(dtype)
    ql = q.QLinear.from_module(lin, weights=q.qint8, activations=q.qint8).cuda()
    x = torch.randn(M, K).to(dtype).cuda()
    ql.input_scale = (x.abs().max() / 127).to(dtype)
    ql.output_scale = torch.tensor(0.05, dtype=dtype, device="cuda")
    ql.freeze()
    with torch.no_grad():
        y = ql(x)
    xs = torch_to_f32(ql.input_scale)
    xq = O.quantize_symmetric(torch_to_f32(x), tag, "int8", xs)
    ws = O.round_to(torch_to_f32(ql.weight._scale).reshape(-1) * xs, tag)  # input._scale * other._scale in dtype
    acc = O.to_f32(O.qbytes_int_mm(xq, ql.weight._data.cpu().numpy(), ws, tag), tag)
    yq = O.quantize_symmetric(acc, tag, "int8", torch_to_f32(ql.output_scale))
    assert np.array_equal(y._data.cpu().numpy(), yq)


def test_weight_qbytes_tensor_fp8_and_to():
    torch.manual_seed(1)
    w = (torch.randn(64, 128) * 0.1).half().cuda()
    scale = q.AbsmaxOptimizer()(w, qtype=q.qfloat8_e4m3fn, axis=0)
    qw = q.quantize_weight(w, qtype=q.qfloat8_e4m3fn, axis=0, scale=scale)
    assert qw._data.dtype == torch.float8_e4m3fn
    ref = O.quantize_symmetric(torch_to_f32(w), "f16", "e4m3fn", torch_to_f32(scale))
    assert np.array_equal(torch_to_bits(qw._data), ref)
    x = torch.randn(8, 128).half().cuda()
    y = torch.nn.functional.linear(x, qw)
    y64, _ = O.qbytes_mm(torch_to_f32(x), O.fp8_bits_to_f32(ref, "e4m3fn"), torch_to_f32(scale).reshape(-1), "f16")
    assert np.allclose(torch_to_f32(y), y64, rtol=2e-3, atol=1e-3)
    t = qw.t()
    assert t.shape == (128, 64) and t.axis == -1


@pytest.mark.gpu
def test_column_parallel_two_gpus_fused_and_nccl():
    """2-rank column-parallel QLinear on one box: NCCL all-gather path and the all-gather fused into the GEMM epilogue
    (peer stores) both reproduce the single-GPU result (tools/check_tp.py under torchrun)."""
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29533", os.path.join(root, "tools", "check_tp.py")]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "TP CHECK OK" in res.stdout, res.stdout[-2000:]


# ------------------------------------------------- fused output quantisation (SURVEY 8f rank 2)
def _rand8(kind, shape, g):
    if kind == "int8":
        return torch.randint(-127, 128, shape, dtype=torch.int8, generator=g)
    dt = torch.float8_e4m3fn if kind == "e4m3fn" else torch.float8_e5m2
    return (torch.randn(shape, generator=g) * 2).to(dt)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("kind,out_dt", [("int8", torch.int8), ("e4m3fn", torch.float8_e4m3fn), ("int8", torch.float8_e4m3fn),
                                         ("e4m3fn", torch.float8_e5m2)])
@pytest.mark.parametrize("M,N,K", [(64, 256, 128), (300, 512, 1024), (257, 300, 256), (1000, 1024, 512), (8, 48, 64)])
@pytest.mark.parametrize("with_bias", [False, True])
def test_qbytes_linear_quantized_is_the_composition(dtype, kind, out_dt, M, N, K, with_bias):
    """One launch == qbytes_mm (+ bias) followed by quantize_symmetric, bit for bit; both tile heights (128 rows for
    M > 64, 64 rows below), ragged N (element-wise stores), every scale dtype."""
    from quanto_b200 import _native as n
    g = torch.Generator().manual_seed(M * 7 + N + K)
    a = _rand8(kind, (M, K), g).cuda()
    w = _rand8(kind, (N, K), g).cuda()
    scales = ((torch.rand(N, 1, generator=g) + 0.5) * (2e-4 if kind == "int8" else 2e-2)).to(dtype).cuda()
    bias = torch.randn(N, generator=g).to(dtype).cuda() if with_bias else None
    y = torch.ops.quanto.qbytes_linear(a, w, scales, bias)
    out_scale = (y.float().abs().max() / (100.0 if out_dt == torch.int8 else 300.0)).to(dtype)
    ref = torch.ops.quanto.quantize_symmetric(y, out_dt, None, out_scale)
    got = torch.ops.quanto.qbytes_linear_quantized(a, w, scales, bias, out_scale, out_dt)
    assert got.dtype == out_dt and got.shape == (M, N)
    assert torch.equal(got.view(torch.uint8), ref.view(torch.uint8)), float((got.view(torch.uint8) != ref.view(torch.uint8)).float().mean())
    # and it really was the fused kernel (status 0 from the C entry point, wgmma family)
    lib = n.load()
    out = torch.empty((M, N), dtype=out_dt, device="cuda")
    rc = lib.qb200_qbytes_mm_quantized(n.ptr(a), n.ptr(w), n.ptr(scales.reshape(-1).contiguous()), n.ptr(bias), n.ptr(out),
                                       n.ptr(out_scale.reshape(1)), M, N, K, n.DTYPE_CODE[a.dtype], n.DTYPE_CODE[w.dtype],
                                       n.DTYPE_CODE[dtype], n.DTYPE_CODE[out_dt], n.stream_ptr(a.device))
    assert rc == 0 and lib.qb200_last_kernel_family() == 1
    assert torch.equal(out.view(torch.uint8), ref.view(torch.uint8))


def test_qbytes_linear_quantized_unsupported_falls_back_to_native_composition():
    from quanto_b200 import _native as n
    g = torch.Generator().manual_seed(0)
    a = _rand8("int8", (16, 40), g).cuda()  # K % 16 != 0: no tensor-core kernel
    w = _rand8("int8", (24, 40), g).cuda()
    scales = (torch.rand(24, 1, generator=g) * 1e-3).to(torch.bfloat16).cuda()
    out_scale = torch.tensor(0.01, dtype=torch.bfloat16, device="cuda")
    lib = n.load()
    out = torch.empty((16, 24), dtype=torch.int8, device="cuda")
    rc = lib.qb200_qbytes_mm_quantized(n.ptr(a), n.ptr(w), n.ptr(scales), None, n.ptr(out), n.ptr(out_scale), 16, 24, 40,
                                       n.I8, n.I8, n.BF16, n.I8, n.stream_ptr(a.device))
    assert rc == 2  # QB200_ERR_UNSUPPORTED
    got = torch.ops.quanto.qbytes_linear_quantized(a, w, scales, None, out_scale, torch.int8)
    ref = torch.ops.quanto.quantize_symmetric(torch.ops.quanto.qbytes_mm(a, w, scales), torch.int8, None, out_scale)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("aq", [q.qint8, q.qfloat8_e4m3fn])
def test_qlinear_quantized_in_and_out_single_launch_chain(with_bias, aq):
    """QLinear(weights=qint8 / qfloat8, activations=same): input quantisation, linear (+ bias) and output quantisation
    vs the oracle chain, bit-exact for int8; the fused forward and the hook-by-hook path agree for both."""
    torch.manual_seed(5)
    K, N, M = 512, 384, 200
    dtype, tag = torch.bfloat16, "bf16"
    lin = torch.nn.Linear(K, N, bias=with_bias).to(dtype)
    wq = q.qint8 if aq == q.qint8 else q.qfloat8_e4m3fn
    ql = q.QLinear.from_module(lin, weights=wq, activations=aq).cuda()
    x = torch.randn(M, K).to(dtype).cuda()
    qmax = 127.0 if aq == q.qint8 else 448.0
    ql.input_scale = (x.abs().max() / qmax).to(dtype)
    ql.output_scale = torch.tensor(0.02 if aq == q.qint8 else 0.005, dtype=dtype, device="cuda")
    ql.freeze()
    with torch.no_grad():
        y = ql(x)  # fused: quantize_input (1 launch) + scales product + ONE linear/bias/quantize_output launch
        assert isinstance(y, q.ActivationQBytesTensor) and y.qtype == aq and y._data.dtype == aq.dtype
        xq = q.quantize_activation(x, aq, ql.input_scale)
        y_float = torch.nn.functional.linear(xq, ql.weight, ql.bias)  # the reference's sequence, op by op
        y_hook = q.quantize_activation(y_float, aq, ql.output_scale)
    assert torch.equal(y._data.view(torch.uint8), y_hook._data.view(torch.uint8))
    assert torch.equal(y._scale, ql.output_scale)
    if aq == q.qint8:
        xs = torch_to_f32(ql.input_scale)
        xq_o = O.quantize_symmetric(torch_to_f32(x), tag, "int8", xs)
        ws = O.round_to(torch_to_f32(ql.weight._scale).reshape(-1) * xs, tag)
        acc = O.to_f32(O.qbytes_int_mm(xq_o, ql.weight._data.cpu().numpy(), ws, tag), tag)
        if with_bias:
            acc = O.round_to(acc + torch_to_f32(ql.bias), tag)
        yq = O.quantize_symmetric(acc, tag, "int8", torch_to_f32(ql.output_scale))
        assert np.array_equal(y._data.cpu().numpy(), yq)
    # without the output hook the forward returns floats again
    ql.disable_output_quantization()
    with torch.no_grad():
        y2 = ql(x)
    assert not isinstance(y2, q.ActivationQBytesTensor) and torch.equal(y2, y_float)
