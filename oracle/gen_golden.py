"""Generate golden vectors from the REAL reference (huggingface/optimum-quanto, CPU path).

Run in the authoring container only (the reference cannot travel to the GPU box):

    PYTHONPATH=/root/reference python oracle/gen_golden.py

It imports `optimum.quanto` from /root/reference, runs the reference's own entry points
(SURVEY.md section 8c) on seeded inputs and writes small `.npz` fixtures to tests/golden/.
bf16 / fp16 / fp8 tensors are stored as raw bit patterns (uint16 / uint8).

The fixtures pin oracle/quanto_oracle.py (tests/test_oracle_golden.py) and are replayed
against the CUDA kernels through the C-ABI (tests/test_gpu_golden.py).
"""
import os
import sys

import numpy as np
import torch

import optimum.quanto  # noqa: F401  (registers torch.ops.quanto.*)
from optimum.quanto import MaxOptimizer, qint2, qint4, qint8, qfloat8_e4m3fn, qfloat8_e4m3fnuz, qfloat8_e5m2
from optimum.quanto.tensor.packed import pack_weights
from optimum.quanto.tensor.weights import quantize_weight

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden")
os.makedirs(OUT, exist_ok=True)

TAG = {torch.float32: "f32", torch.float16: "f16", torch.bfloat16: "bf16"}
F8TAG = {torch.float8_e4m3fn: "e4m3fn", torch.float8_e5m2: "e5m2", torch.float8_e4m3fnuz: "e4m3fnuz"}


def bits(t: torch.Tensor) -> np.ndarray:
    t = t.detach().contiguous()
    if t.dtype == torch.float32:
        return t.numpy()
    if t.dtype in (torch.float16, torch.bfloat16):
        return t.view(torch.int16).numpy().view(np.uint16)
    if t.dtype in F8TAG:
        return t.view(torch.uint8).numpy()
    return t.numpy()


def gen_unpack(g):
    cases = {}
    for i, (shape, nbits) in enumerate(
        [((12,), 4), ((32, 32), 4), ((10, 16), 4), ((12,), 2), ((32, 32), 2), ((7, 48), 2), ((256, 128), 4)]
    ):
        packed = torch.randint(0, 256, shape, dtype=torch.uint8, generator=g)
        out = torch.ops.quanto.unpack(packed, nbits)
        cases[f"c{i}_bits"] = np.int64(nbits)
        cases[f"c{i}_in"] = packed.numpy()
        cases[f"c{i}_out"] = out.numpy()
    # pack_weights incl. odd row counts (tests/tensor/test_packed_tensor.py:24-35)
    for i, (shape, nbits) in enumerate([((10, 8), 4), ((12, 8), 4), ((10,), 2), ((13, 4), 2), ((64, 128), 4)]):
        u = torch.randint(0, 2 ** nbits, shape, dtype=torch.uint8, generator=g)
        cases[f"p{i}_bits"] = np.int64(nbits)
        cases[f"p{i}_in"] = u.numpy()
        cases[f"p{i}_out"] = pack_weights(u, nbits).numpy()
    cases["n_unpack"] = np.int64(7)
    cases["n_pack"] = np.int64(5)
    np.savez_compressed(os.path.join(OUT, "unpack.npz"), **cases)


def gen_quantize_symmetric(g):
    cases = {}
    idx = 0
    for in_dtype in (torch.float32, torch.float16, torch.bfloat16):
        for out_dtype in (torch.int8, torch.float8_e4m3fn, torch.float8_e5m2):
            for axis, shape in ((None, (37, 64)), (0, (48, 96)), (-1, (48, 96)), (None, (3, 5, 32))):
                base = (torch.rand(shape, generator=g) * 2 - 1).to(in_dtype) * 3
                if axis is None:
                    scale = (base.abs().max().float() / 100).to(in_dtype)
                elif axis == 0:
                    scale = (base.abs().amax(dim=1, keepdim=True).float() / 127).to(in_dtype)
                else:
                    scale = (base.abs().amax(dim=0, keepdim=True).float() / 127).to(in_dtype)
                out = torch.ops.quanto.quantize_symmetric(base, dtype=out_dtype, axis=axis, scale=scale)
                p = f"c{idx}_"
                cases[p + "in_tag"] = np.array(TAG[in_dtype])
                cases[p + "out_tag"] = np.array("int8" if out_dtype == torch.int8 else F8TAG[out_dtype])
                cases[p + "axis"] = np.int64(-2 if axis is None else axis)
                cases[p + "base"] = bits(base)
                cases[p + "scale"] = bits(scale)
                cases[p + "out"] = bits(out)
                idx += 1
    cases["n"] = np.int64(idx)
    np.savez_compressed(os.path.join(OUT, "quantize_symmetric.npz"), **cases)


def gen_qbits(g):
    """int4/int2 weights: canonical storage, dequantize() and F.linear through the python path (optimized=False)."""
    cases = {}
    idx = 0
    cfgs = [
        # (dtype, qtype, N, K, group, M, zeropoint, bias)
        (torch.bfloat16, qint4, 256, 256, 128, 16, False, False),
        (torch.bfloat16, qint4, 128, 512, 128, 33, False, True),
        (torch.float16, qint4, 256, 256, 128, 16, False, False),
        (torch.float16, qint4, 128, 384, 128, 8, False, True),
        (torch.bfloat16, qint4, 128, 256, 128, 1, True, False),
        (torch.float16, qint4, 128, 256, 128, 5, True, False),
        (torch.bfloat16, qint4, 64, 256, 64, 4, False, False),
        (torch.float32, qint4, 64, 256, 128, 4, False, False),
        (torch.bfloat16, qint2, 64, 256, 128, 4, False, False),
    ]
    for dtype, qt, N, K, G, M, zeropoint, with_bias in cfgs:
        W = (torch.randn(N, K, generator=g) * 0.02).to(dtype)
        scale, shift = MaxOptimizer()(W, qtype=qt, axis=0, group_size=G, zeropoint=zeropoint)
        qW = quantize_weight(W, qtype=qt, axis=0, scale=scale, shift=shift, group_size=G, optimized=False)
        x = torch.randn(M, K, generator=g).to(dtype)
        bias = torch.randn(N, generator=g).to(dtype) if with_bias else None
        y = torch.nn.functional.linear(x, qW, bias)
        deq = qW.dequantize()
        p = f"c{idx}_"
        cases[p + "tag"] = np.array(TAG[dtype])
        cases[p + "bits"] = np.int64(qt.bits)
        cases[p + "shape"] = np.array([N, K, G, M], dtype=np.int64)
        cases[p + "zeropoint"] = np.int64(int(zeropoint))
        cases[p + "packed"] = qW._data._data.numpy()
        cases[p + "scale"] = bits(qW._scale)
        cases[p + "shift"] = bits(qW._shift)
        cases[p + "x"] = bits(x)
        if bias is not None:
            cases[p + "bias"] = bits(bias)
        cases[p + "deq"] = bits(deq)
        cases[p + "y"] = bits(y)
        idx += 1
    cases["n"] = np.int64(idx)
    np.savez_compressed(os.path.join(OUT, "qbits.npz"), **cases)


def gen_qbytes(g):
    """torch.ops.quanto.qbytes_mm on CPU tensors (dispatch library/qbytes_mm.py:91-105)."""
    cases = {}
    idx = 0
    # (A kind, W kind, out dtype, M, K, N)
    cfgs = [
        ("int8", "int8", torch.bfloat16, 32, 64, 48),
        ("int8", "int8", torch.float16, 24, 128, 64),
        ("int8", "int8", torch.float32, 8, 32, 48),
        ("int8", "int8", torch.bfloat16, 256, 1024, 1024),  # BASELINE cfg1 shape, int8 activations
        ("same", "int8", torch.float32, 16, 64, 48),
        ("same", "int8", torch.float16, 10, 50, 50),
        ("same", "int8", torch.bfloat16, 10, 32, 64),  # NB: CPU routes bf16 x int8 (K%4==0) to _weight_int8pack_mm
        ("same", "e4m3fn", torch.float16, 16, 64, 48),
        ("same", "e4m3fn", torch.bfloat16, 16, 64, 48),
        ("same", "e5m2", torch.bfloat16, 16, 64, 48),
        ("e4m3fn", "e4m3fn", torch.bfloat16, 16, 64, 48),
        ("e4m3fn", "e4m3fn", torch.float16, 32, 128, 64),
        ("e4m3fn", "int8", torch.bfloat16, 16, 64, 48),
        ("e5m2", "e4m3fn", torch.float16, 16, 64, 48),
    ]
    f8 = {"e4m3fn": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}
    for akind, wkind, odt, M, K, N in cfgs:
        if akind == "int8":
            A = torch.randint(-127, 127, (M, K), dtype=torch.int8, generator=g)
        elif akind == "same":
            A = (torch.rand(M, K, generator=g) * 2 - 1).to(odt)
        else:
            A = (torch.randn(M, K, generator=g)).clamp(-400, 400).to(f8[akind])
        if wkind == "int8":
            W = torch.randint(-127, 127, (N, K), dtype=torch.int8, generator=g)
        else:
            W = (torch.randn(N, K, generator=g) * 2).to(f8[wkind])
        scales = (torch.rand(N, 1, generator=g) / 1e3 + 1e-5).to(odt)
        y = torch.ops.quanto.qbytes_mm(A, W, scales)
        p = f"c{idx}_"
        cases[p + "akind"] = np.array(akind)
        cases[p + "wkind"] = np.array(wkind)
        cases[p + "tag"] = np.array(TAG[odt])
        cases[p + "A"] = bits(A)
        cases[p + "W"] = bits(W)
        cases[p + "scales"] = bits(scales)
        cases[p + "y"] = bits(y)
        idx += 1
    cases["n"] = np.int64(idx)
    np.savez_compressed(os.path.join(OUT, "qbytes_mm.npz"), **cases)


def gen_qlinear(g):
    """QLinear end to end (nn/qlinear.py:49-50): weights qint8/qint4/qfloat8, activations None/qint8, frozen."""
    from optimum.quanto import Calibration, freeze, quantize  # noqa: F401
    from optimum.quanto.nn import QLinear

    cases = {}
    idx = 0
    for dtype, wq, aq, K, N, M in [
        (torch.bfloat16, qint8, None, 1024, 1024, 256),  # BASELINE configs[0]
        (torch.float16, qint8, qint8, 128, 64, 32),
        (torch.bfloat16, qint4, None, 256, 128, 16),
        (torch.float16, qfloat8_e4m3fn, None, 128, 64, 8),
        (torch.bfloat16, qint8, qfloat8_e4m3fn, 128, 64, 32),
    ]:
        lin = torch.nn.Linear(K, N, bias=True).to(dtype)
        with torch.no_grad():
            lin.weight.copy_((torch.randn(N, K, generator=g) * 0.05).to(dtype))
            lin.bias.copy_((torch.randn(N, generator=g) * 0.1).to(dtype))
        q = QLinear.from_module(lin, weights=wq, activations=aq)
        x = torch.randn(M, K, generator=g).to(dtype)
        if aq is not None:
            q.input_scale = (x.abs().max().float() / (127.0 if aq == qint8 else 448.0)).to(dtype)
            with torch.no_grad():
                y_float = lin(x)
            q.output_scale = (y_float.abs().max().float() / (127.0 if aq == qint8 else 448.0)).to(dtype)
        # freeze WITHOUT the device-specific repacking: keep canonical tensors (optimized=False route)
        qw = q.qweight
        if type(qw).__name__ not in ("WeightQBytesTensor", "WeightQBitsTensor"):
            if hasattr(qw, "weight_qbits_tensor"):
                qw = qw.weight_qbits_tensor()
            else:
                qw = qw.weight_qbytes_tensor()
        q.weight = torch.nn.Parameter(qw)
        with torch.no_grad():
            y = q(x)
        p = f"c{idx}_"
        cases[p + "tag"] = np.array(TAG[dtype])
        cases[p + "wq"] = np.array(wq.name)
        cases[p + "aq"] = np.array("none" if aq is None else aq.name)
        cases[p + "x"] = bits(x)
        cases[p + "bias"] = bits(lin.bias)
        cases[p + "input_scale"] = bits(q.input_scale.reshape(1))
        cases[p + "output_scale"] = bits(q.output_scale.reshape(1))
        sd = q.state_dict()
        for k, v in sd.items():
            if k.startswith("weight"):
                cases[p + "sd_" + k] = bits(v)
        cases[p + "shape"] = np.array([N, K, M, q.weight_group_size or 0], dtype=np.int64)
        if aq is None:
            cases[p + "y"] = bits(y)
        else:
            cases[p + "y_data"] = bits(y._data)
            cases[p + "y_scale"] = bits(y._scale.reshape(1))
        idx += 1
    cases["n"] = np.int64(idx)
    np.savez_compressed(os.path.join(OUT, "qlinear.npz"), **cases)


def gen_freeze(g):
    """Weight freeze (SURVEY 8f): MaxOptimizer + quanto::quantize_affine + pack_weights, AbsmaxOptimizer +
    quanto::quantize_symmetric, through the reference's own entry points on CPU tensors."""
    from optimum.quanto import AbsmaxOptimizer

    cases = {}
    idx = 0
    # (dtype, qtype, N, K, group (None = per-axis), zeropoint)
    cfgs = [
        (torch.bfloat16, qint4, 64, 256, 128, False),
        (torch.bfloat16, qint4, 64, 256, 128, True),
        (torch.float16, qint4, 32, 384, 128, False),
        (torch.float16, qint4, 32, 192, 64, True),
        (torch.float32, qint4, 32, 256, 128, False),
        (torch.float32, qint4, 16, 96, 32, True),
        (torch.bfloat16, qint2, 64, 256, 128, False),
        (torch.float16, qint2, 36, 128, 32, True),
        (torch.bfloat16, qint4, 33, 96, 96, False),   # odd number of grouped rows, 96-wide groups
        (torch.bfloat16, qint4, 48, 64, None, False),  # per-axis (K <= 128): rows = N
        (torch.bfloat16, qint2, 27, 64, None, False),  # rows not a multiple of 4
    ]
    for dtype, qt, N, K, G, zeropoint in cfgs:
        W = (torch.randn(N, K, generator=g) * 0.02).to(dtype)
        scale, shift = MaxOptimizer()(W, qtype=qt, axis=0, group_size=G, zeropoint=zeropoint)
        data = torch.ops.quanto.quantize_affine(W, qt.bits, 0, G, scale, shift)
        qW = quantize_weight(W, qtype=qt, axis=0, scale=scale, shift=shift, group_size=G, optimized=False)
        assert torch.equal(qW._data.unpack(), data)
        p = f"a{idx}_"
        cases[p + "tag"] = np.array(TAG[dtype])
        cases[p + "bits"] = np.int64(qt.bits)
        cases[p + "shape"] = np.array([N, K, G or 0], dtype=np.int64)
        cases[p + "zeropoint"] = np.int64(int(zeropoint))
        cases[p + "W"] = bits(W)
        cases[p + "scale"] = bits(scale)
        cases[p + "shift"] = bits(shift)
        cases[p + "data"] = data.numpy()
        cases[p + "packed"] = qW._data._data.numpy()
        idx += 1
    cases["n_affine"] = np.int64(idx)
    idx = 0
    for dtype, qt, N, K in [
        (torch.bfloat16, qint8, 48, 256),
        (torch.float16, qint8, 32, 100),
        (torch.float32, qint8, 16, 64),
        (torch.bfloat16, qfloat8_e4m3fn, 32, 128),
        (torch.float16, qfloat8_e5m2, 32, 128),
        (torch.bfloat16, qint8, 8, 8200),
    ]:
        W = (torch.randn(N, K, generator=g) * 0.05).to(dtype)
        scale = AbsmaxOptimizer()(W, qtype=qt, axis=0)
        scale_t = AbsmaxOptimizer()(W, qtype=qt, axis=None)
        data = torch.ops.quanto.quantize_symmetric(W, dtype=qt.dtype, axis=0, scale=scale)
        p = f"s{idx}_"
        cases[p + "tag"] = np.array(TAG[dtype])
        cases[p + "out_tag"] = np.array("int8" if qt.dtype == torch.int8 else F8TAG[qt.dtype])
        cases[p + "qmax"] = np.float64(qt.qmax)
        cases[p + "W"] = bits(W)
        cases[p + "scale"] = bits(scale)
        cases[p + "scale_tensor"] = bits(scale_t.reshape(1))
        cases[p + "data"] = bits(data)
        idx += 1
    cases["n_absmax"] = np.int64(idx)
    np.savez_compressed(os.path.join(OUT, "freeze.npz"), **cases)


def gen_affine_zp(g):
    """quanto::quantize_affine with INTEGER shifts taken by value (library/quantize.py:74-76): int8 zero-points built the way
    the reference's own test builds them -- torch.round(shift / scale).to(torch.int8), negative for groups whose minimum is
    positive (tests/tensor/weights/test_weight_qbits_tensor_quantize.py:37-39) -- and uint8 ones beyond the quantized
    range.  A separate file: the fixtures committed earlier stay byte-identical."""
    cases = {}
    idx = 0
    for dtype in (torch.float32, torch.float16, torch.bfloat16):
        for axis, shape, G in ((0, (32, 64), 16), (-1, (32, 32), 8), (-1, (32, 10, 32), 8), (0, (24, 96), 32)):
            for zdtype in (torch.int8, torch.uint8):
                base = (torch.rand(shape, generator=g) * 2 - 1 + 0.8).to(dtype)  # many groups lie entirely above zero
                scale, shift = MaxOptimizer()(base, qtype=qint4, axis=axis, group_size=G)
                if zdtype == torch.int8:
                    zp = torch.round(shift / scale).to(torch.int8)
                else:
                    zp = torch.randint(0, 60, shift.shape, generator=g).to(torch.uint8)
                data = torch.ops.quanto.quantize_affine(base, 4, axis, G, scale, zp)
                p = f"z{idx}_"
                cases[p + "tag"] = np.array(TAG[dtype])
                cases[p + "axis"] = np.int64(axis)
                cases[p + "shape"] = np.array(list(shape), dtype=np.int64)
                cases[p + "group"] = np.int64(G)
                cases[p + "base"] = bits(base)
                cases[p + "scale"] = bits(scale)
                cases[p + "zp"] = zp.numpy()
                cases[p + "data"] = data.numpy()
                idx += 1
    cases["n"] = np.int64(idx)
    np.savez_compressed(os.path.join(OUT, "affine_zp.npz"), **cases)


def gen_fnuz(g):
    """float8_e4m3fnuz (bias 8, max 240, 0x80 = NaN, no negative zero) through the reference's own entry points:
    quantize_symmetric to it (all-zero rows, quotients past +-240, tiny negatives), qbytes_mm with e4m3fnuz weights
    (the reference's tests/library/test_mm.py "w-float8-uz" cases) and two frozen QLinear layers.  A separate file with
    its own seed: the fixtures committed earlier stay byte-identical."""
    from optimum.quanto.nn import QLinear

    fnuz = torch.float8_e4m3fnuz
    cases = {}
    idx = 0
    for in_dtype in (torch.float32, torch.float16, torch.bfloat16):
        for axis, shape in ((None, (37, 64)), (0, (48, 96)), (-1, (48, 96))):
            base = (torch.rand(shape, generator=g) * 2 - 1) * 3
            base[:, :4] *= 1e-5  # |quotient| below half the smallest subnormal (2^-11): +-0 -> 0x00, never 0x80
            if axis is None:
                base = base.to(in_dtype)
                scale = (base.abs().max().float() / 300).to(in_dtype)  # quotients up to +-300: clamped to +-240
            elif axis == 0:
                base[5] = 0  # all-zero row: scale 0, quotient 0/0 -> NaN -> 0x80
                base = base.to(in_dtype)
                scale = (base.abs().amax(dim=1, keepdim=True).float() / 240).to(in_dtype)
            else:
                base = base.to(in_dtype)
                scale = (base.abs().amax(dim=0, keepdim=True).float() / 260).to(in_dtype)
            out = torch.ops.quanto.quantize_symmetric(base, dtype=fnuz, axis=axis, scale=scale)
            p = f"q{idx}_"
            cases[p + "in_tag"] = np.array(TAG[in_dtype])
            cases[p + "axis"] = np.int64(-2 if axis is None else axis)
            cases[p + "base"] = bits(base)
            cases[p + "scale"] = bits(scale)
            cases[p + "out"] = bits(out)
            idx += 1
    cases["n_quantize"] = np.int64(idx)
    idx = 0
    # (activation kind, out dtype, M, K, N): "same" = activations in the output dtype
    for akind, odt, M, K, N in [
        ("same", torch.float16, 32, 32, 48),
        ("same", torch.bfloat16, 32, 64, 50),
        ("same", torch.float16, 10, 80, 64),
        ("same", torch.bfloat16, 10, 80, 48),
        ("f32", torch.bfloat16, 16, 64, 48),
        ("int8", torch.float16, 32, 50, 64),
        ("int8", torch.bfloat16, 10, 64, 50),
        ("e4m3fnuz", torch.float16, 16, 64, 48),
    ]:
        if akind == "int8":
            A = torch.randint(-127, 127, (M, K), dtype=torch.int8, generator=g)
        elif akind == "e4m3fnuz":
            A = torch.randn(M, K, generator=g).to(fnuz)
        else:
            A = (torch.rand(M, K, generator=g) * 2 - 1).to(odt if akind == "same" else torch.float32)
        W = (torch.randn(N, K, generator=g) * 20).clamp(-240, 240).to(fnuz)
        scales = (torch.rand(N, 1, generator=g) / 1e3 + 1e-5).to(odt)
        y = torch.ops.quanto.qbytes_mm(A, W, scales)
        p = f"m{idx}_"
        cases[p + "akind"] = np.array(akind)
        cases[p + "tag"] = np.array(TAG[odt])
        cases[p + "A"] = bits(A)
        cases[p + "W"] = bits(W)
        cases[p + "scales"] = bits(scales)
        cases[p + "y"] = bits(y)
        idx += 1
    cases["n_mm"] = np.int64(idx)
    idx = 0
    for dtype, wq, aq, K, N, M in [
        (torch.float16, qfloat8_e4m3fnuz, None, 128, 64, 8),
        (torch.bfloat16, qint8, qfloat8_e4m3fnuz, 128, 64, 32),
    ]:
        lin = torch.nn.Linear(K, N, bias=True).to(dtype)
        with torch.no_grad():
            lin.weight.copy_((torch.randn(N, K, generator=g) * 0.05).to(dtype))
            lin.bias.copy_((torch.randn(N, generator=g) * 0.1).to(dtype))
        q = QLinear.from_module(lin, weights=wq, activations=aq)
        x = torch.randn(M, K, generator=g).to(dtype)
        if aq is not None:
            q.input_scale = (x.abs().max().float() / 240.0).to(dtype)
            with torch.no_grad():
                y_float = lin(x)
            q.output_scale = (y_float.abs().max().float() / 240.0).to(dtype)
        qw = q.qweight  # canonical tensors, as in gen_qlinear
        if type(qw).__name__ != "WeightQBytesTensor":
            qw = qw.weight_qbytes_tensor()
        q.weight = torch.nn.Parameter(qw)
        with torch.no_grad():
            y = q(x)
        p = f"l{idx}_"
        cases[p + "tag"] = np.array(TAG[dtype])
        cases[p + "wq"] = np.array(wq.name)
        cases[p + "aq"] = np.array("none" if aq is None else aq.name)
        cases[p + "x"] = bits(x)
        cases[p + "bias"] = bits(lin.bias)
        cases[p + "input_scale"] = bits(q.input_scale.reshape(1))
        cases[p + "output_scale"] = bits(q.output_scale.reshape(1))
        for k, v in q.state_dict().items():
            if k.startswith("weight"):
                cases[p + "sd_" + k] = bits(v)
        cases[p + "shape"] = np.array([N, K, M, 0], dtype=np.int64)
        if aq is None:
            cases[p + "y"] = bits(y)
        else:
            cases[p + "y_data"] = bits(y._data)
            cases[p + "y_scale"] = bits(y._scale.reshape(1))
        idx += 1
    cases["n_qlinear"] = np.int64(idx)
    np.savez_compressed(os.path.join(OUT, "fnuz.npz"), **cases)


def main():
    torch.set_num_threads(1)  # deterministic accumulation order for the stored float results
    if "--affine-zp-only" in sys.argv:  # added in round 2 (a bug found by the reference's own tests): new file only
        gen_affine_zp(torch.Generator().manual_seed(20260924))
        return 0
    if "--fnuz-only" in sys.argv:  # added with the float8_e4m3fnuz coverage: new file only
        gen_fnuz(torch.Generator().manual_seed(20261017))
        return 0
    if "--freeze-only" in sys.argv:  # added after the first fixtures were committed: keeps those byte-identical
        gen_freeze(torch.Generator().manual_seed(20260923))
        return 0
    g = torch.Generator().manual_seed(20260922)
    gen_unpack(g)
    gen_quantize_symmetric(g)
    gen_qbits(g)
    gen_qbytes(g)
    gen_qlinear(g)
    gen_freeze(torch.Generator().manual_seed(20260923))
    gen_affine_zp(torch.Generator().manual_seed(20260924))
    gen_fnuz(torch.Generator().manual_seed(20261017))
    tot = sum(os.path.getsize(os.path.join(OUT, f)) for f in os.listdir(OUT))
    print("wrote fixtures to", os.path.normpath(OUT), f"({tot/1024:.0f} KiB)")


if __name__ == "__main__":
    sys.exit(main())
