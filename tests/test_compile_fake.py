"""Fake (meta) implementations of every `torch.ops.quanto.*` op: the metadata torch.compile / AOTAutograd trace with.

CPU only: fake CUDA tensors need no device.  Each case states the shape, dtype and strides the CUDA implementation in
library.py allocates for those arguments.
"""
import os
import re
import subprocess
import sys

import pytest
import torch
from torch._dynamo.source import ConstantSource
from torch._subclasses.fake_tensor import FakeTensorMode
from torch.fx.experimental.symbolic_shapes import ShapeEnv

import quanto_b200  # noqa: F401  (registers the ops)
from quanto_b200 import library

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBRARY_PY = os.path.join(ROOT, "optimum-quanto_b200", "quanto_b200", "library.py")
BF16, F16, F32, U8, I8 = torch.bfloat16, torch.float16, torch.float32, torch.uint8, torch.int8
E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
Q = torch.ops.quanto


def defined_ops():
    """Every op name library.py defines (parsed from its source, so that a new op cannot go without a fake)."""
    with open(LIBRARY_PY) as f:
        return re.findall(r'^_define\("(\w+)"', f.read(), flags=re.M)


def contiguous_strides(shape):
    strides, acc = [], 1
    for d in reversed(shape):
        strides.append(acc)
        acc *= d
    return tuple(reversed(strides))


def e(*shape, dtype=BF16):
    return torch.empty(shape, dtype=dtype, device="cuda")


def check(out, shape, dtype):
    assert tuple(out.shape) == tuple(shape)
    assert out.dtype == dtype
    assert out.device.type == "cuda"
    assert out.stride() == contiguous_strides(shape)


# (op name, argument builder, [(expected shape, dtype), ...] for each output)
CASES = [
    ("unpack", lambda: (e(64, 32, dtype=U8), 4), [((128, 32), U8)]),
    ("unpack", lambda: (e(7, 16, dtype=U8), 2), [((28, 16), U8)]),
    ("pack", lambda: (e(128, 32, dtype=U8), 4), [((64, 32), U8)]),
    ("pack", lambda: (e(129, 32, dtype=U8), 4), [((65, 32), U8)]),
    ("pack", lambda: (e(130, 16, dtype=I8), 2), [((33, 16), U8)]),
    ("quantize_symmetric", lambda: (e(4, 3, 64), I8, None, e()), [((4, 3, 64), I8)]),
    ("quantize_symmetric", lambda: (e(32, 64, dtype=F16), E4M3, 0, e(32, 1, dtype=F16)), [((32, 64), E4M3)]),
    ("quantize_symmetric", lambda: (e(32, 64), E5M2, -1, e(1, 64)), [((32, 64), E5M2)]),
    ("quantize_affine", lambda: (e(32, 256), 4, 0, 128, e(64, 1), e(64, 1, dtype=U8)), [((64, 128), U8)]),
    ("quantize_affine", lambda: (e(32, 256), 2, 0, None, e(32, 1), e(32, 1)), [((32, 256), U8)]),
    ("quantize_qbits_max", lambda: (e(32, 256), 4, 128, False), [((32, 128), U8), ((64, 1), BF16), ((64, 1), BF16)]),
    ("quantize_qbits_max", lambda: (e(3, 64, dtype=F16), 4, 64, True), [((2, 64), U8), ((3, 1), F16), ((3, 1), U8)]),
    ("quantize_qbits_max", lambda: (e(5, 128), 2, 64, True), [((3, 64), U8), ((10, 1), BF16), ((10, 1), U8)]),
    ("quantize_qbits_hqq", lambda: (e(3, 256), 4, 128, False, 0.7, 10.0, 1.01, 20),
     [((3, 128), U8), ((6, 1), BF16), ((6, 1), BF16), ((22,), F32)]),
    ("quantize_qbits_hqq", lambda: (e(8, 64, dtype=F16), 2, 64, True, 0.7, 10.0, 1.01, 0),
     [((2, 64), U8), ((8, 1), F16), ((8, 1), U8), ((2,), F32)]),
    ("hqq_shrink", lambda: (e(7, 33, dtype=F16), 10.0, 0.7), [((7, 33), F16)]),
    ("quantize_qbytes_absmax", lambda: (e(48, 96), I8), [((48, 96), I8), ((48, 1), BF16)]),
    ("quantize_qbytes_absmax", lambda: (e(16, 32, dtype=F16), E4M3), [((16, 32), E4M3), ((16, 1), F16)]),
    ("absmax", lambda: (e(5, 7, 9),), [((), BF16)]),
    ("qbytes_mm", lambda: (e(3, 5, 64), e(96, 64, dtype=I8), e(96, 1, dtype=F16)), [((3, 5, 96), F16)]),
    ("qbytes_mm", lambda: (e(8, 64, dtype=E4M3), e(96, 64, dtype=E4M3), e()), [((8, 96), BF16)]),
    ("qbytes_linear", lambda: (e(2, 4, 64), e(96, 64, dtype=I8), e(96, 1), e(96)), [((2, 4, 96), BF16)]),
    ("qbytes_linear", lambda: (e(4, 64), e(96, 64, dtype=I8), e(96, 1), e(96, dtype=F32)), [((4, 96), F32)]),
    ("qbytes_linear_quantized", lambda: (e(2, 3, 64, dtype=I8), e(96, 64, dtype=I8), e(96, 1), e(96), e(), I8),
     [((2, 3, 96), I8)]),
    ("qbytes_linear_quantized", lambda: (e(5, 64, dtype=E4M3), e(96, 64, dtype=E4M3), e(96, 1), None, e(), E5M2),
     [((5, 96), E5M2)]),
    ("qbytes_linear_quantized", lambda: (e(5, 64, dtype=I8), e(96, 64, dtype=I8), e(96, 1), e(96, dtype=F32), e(), I8),
     [((5, 96), I8)]),
    ("dequantize_qbits", lambda: (e(96, 128, dtype=U8), e(192, 1), e(192, 1, dtype=U8), 96, 256, 128, 4),
     [((96, 256), BF16)]),
    ("dequantize_qbits", lambda: (e(3, 64, dtype=U8), e(10, 1, dtype=F16), e(10, 1, dtype=F16), 5, 128, 64, 2),
     [((5, 128), F16)]),
    ("qbits_mm", lambda: (e(3, 5, 256), e(96, 128, dtype=U8), e(192, 1), e(192, 1), None, 96, 128, 4),
     [((3, 5, 96), BF16)]),
    ("qbits_mm", lambda: (e(7, 256, dtype=F16), e(15, 128, dtype=U8), e(30, 1, dtype=F16),
                          e(30, 1, dtype=U8), e(15, dtype=F16), 15, 128, 4), [((7, 15), F16)]),
    ("qbits_mm", lambda: (e(1, 128), e(2, 128, dtype=U8), e(5, 1), e(5, 1, dtype=U8), e(5), 5, 128, 2),
     [((1, 5), BF16)]),
    ("qbits_grad_input", lambda: (e(16, 96), e(96, 128, dtype=U8), e(192, 1), e(192, 1), 96, 128, 4),
     [((16, 256), BF16)]),
    ("qbits_grad_input", lambda: (e(300, 5, dtype=F16), e(3, 64, dtype=U8), e(10, 1, dtype=F16),
                                  e(10, 1, dtype=U8), 5, 64, 2), [((300, 128), F16)]),
    ("qbytes_grad_input", lambda: (e(16, 96), e(96, 64, dtype=I8), e(96, 1)), [((16, 64), BF16)]),
    ("qbytes_grad_input", lambda: (e(300, 96, dtype=F16), e(96, 64, dtype=E5M2), e(dtype=F16)), [((300, 64), F16)]),
]


@pytest.mark.parametrize("name,args,expected", CASES, ids=[f"{c[0]}-{i}" for i, c in enumerate(CASES)])
def test_fake_matches_cuda_allocation(name, args, expected):
    with FakeTensorMode():
        out = getattr(Q, name)(*args())
    outs = out if isinstance(out, tuple) else (out,)
    assert len(outs) == len(expected)
    for o, (shape, dtype) in zip(outs, expected):
        check(o, shape, dtype)


def test_every_defined_op_is_covered_by_a_case():
    assert set(defined_ops()) == {c[0] for c in CASES}


def test_every_defined_op_has_a_fake():
    names = defined_ops()
    assert len(names) == 16 and set(names) == set(library.FAKE_IMPLS)
    for name in names:
        entry = torch._library.simple_registry.singleton.find("quanto::" + name)
        assert entry.fake_impl.kernel is not None, name


def test_fake_checks_are_the_cuda_checks():
    """The fakes reject what the CUDA implementations reject, with the same message."""
    with FakeTensorMode():
        with pytest.raises(ValueError, match="bias must have one value per output feature"):
            Q.qbits_mm(e(4, 256), e(96, 128, dtype=U8), e(192, 1), e(192, 1), e(95), 96, 128, 4)
        with pytest.raises(ValueError, match="does not match the activations"):
            Q.qbits_mm(e(4, 256, dtype=F16), e(96, 128, dtype=U8), e(192, 1), e(192, 1), None, 96, 128, 4)
        with pytest.raises(ValueError, match="in_features mismatch"):
            Q.qbytes_mm(e(4, 63), e(96, 64, dtype=I8), e(96, 1))
        with pytest.raises(ValueError, match="grad_output must be"):
            Q.qbytes_grad_input(e(4, 95), e(96, 64, dtype=I8), e(96, 1))
        with pytest.raises(ValueError, match="Group size"):
            Q.quantize_qbits_max(e(32, 200), 4, 128, False)


def test_fakes_take_symbolic_token_counts():
    """M (tokens) stays a SymInt through the linears and their input gradients."""
    env = ShapeEnv()
    m = env.create_symintnode(env.create_symbol(12, ConstantSource("m")), hint=12)
    assert isinstance(m, torch.SymInt)
    mode = FakeTensorMode(shape_env=env)
    with mode:
        x = torch.empty((m, 256), dtype=BF16, device="cuda")
        y = Q.qbits_mm(x, e(96, 128, dtype=U8), e(192, 1), e(192, 1, dtype=U8), e(96), 96, 128, 4)
        assert y.shape[0] is m or y.shape[0] == m
        assert tuple(y.shape[1:]) == (96,)
        g = Q.qbits_grad_input(y, e(96, 128, dtype=U8), e(192, 1), e(192, 1, dtype=U8), 96, 128, 4)
        assert tuple(g.shape[1:]) == (256,)
        q8 = Q.quantize_symmetric(x, I8, None, e())
        z = Q.qbytes_linear_quantized(q8, e(96, 256, dtype=I8), e(96, 1), e(96), e(), I8)
        assert z.dtype == I8 and tuple(z.shape[1:]) == (96,)
        assert isinstance(z.shape[0], torch.SymInt)


_REFERENCE_FIRST = r"""
import sys
import optimum.quanto  # defines unpack, qbytes_mm, quantize_symmetric and quantize_affine first
import torch
from torch._subclasses.fake_tensor import FakeTensorMode
import quanto_b200
from quanto_b200 import library
for name in library.FAKE_IMPLS:
    assert torch._library.simple_registry.singleton.find("quanto::" + name).fake_impl.kernel is not None, name
with FakeTensorMode():
    a = torch.empty(4, 64, dtype=torch.int8, device="cuda")
    w = torch.empty(96, 64, dtype=torch.int8, device="cuda")
    out = torch.ops.quanto.qbytes_mm(a, w, torch.empty(96, 1, dtype=torch.bfloat16, device="cuda"))
    assert out.shape == (4, 96) and out.dtype == torch.bfloat16
    up = torch.ops.quanto.unpack(torch.empty(7, 16, dtype=torch.uint8, device="cuda"), 4)
    assert up.shape == (14, 16)
print("ok")
"""


def test_fakes_registered_after_reference_import():
    """Same coverage when optimum.quanto defined its four ops before this package was imported."""
    ref = os.path.join(ROOT, "oracle", "_ref")
    path = [p for p in (ref, os.path.join(ROOT, "optimum-quanto_b200"), os.environ.get("PYTHONPATH", "")) if p]
    env = dict(os.environ, PYTHONPATH=os.pathsep.join(path))
    probe = subprocess.run([sys.executable, "-c", "import optimum.quanto"], env=env, capture_output=True, text=True)
    if probe.returncode != 0:
        pytest.skip("the reference package (optimum.quanto) is not importable here")
    run = subprocess.run([sys.executable, "-c", _REFERENCE_FIRST], env=env, capture_output=True, text=True)
    assert run.returncode == 0 and run.stdout.strip().endswith("ok"), run.stderr[-3000:]
