"""CPU checks of the quantized-attention ops: every op library_attention.py defines has a fake that matches the CUDA
allocation, and the attention oracle is pinned to the reference (tests/golden/qattention.npz)."""
import os
import re

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

import quanto_b200  # noqa: F401  (registers the ops)
from quanto_b200 import library_attention
from oracle import attention_oracle as AO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCE = os.path.join(ROOT, "optimum-quanto_b200", "quanto_b200", "library_attention.py")
GOLDEN = os.path.join(ROOT, "tests", "golden", "qattention.npz")
BF16, F16, F32, I8, E4M3 = torch.bfloat16, torch.float16, torch.float32, torch.int8, torch.float8_e4m3fn
Q = torch.ops.quanto


def e(*shape, dtype=BF16):
    return torch.empty(shape, dtype=dtype, device="cuda")


CASES = [
    ("qbytes_bmm", lambda: (e(4, 5, 64, dtype=I8), e(4, 64, 7, dtype=I8), e(), e()), ((4, 5, 7), BF16)),
    ("qbytes_bmm", lambda: (e(2, 3, 10, dtype=I8), e(2, 6, 10, dtype=I8).transpose(1, 2), e(dtype=F32), e(dtype=F32)),
     ((2, 3, 6), F32)),
    ("qbytes_softmax", lambda: (e(2, 3, 50, dtype=I8), e(dtype=F16), e(dtype=F16)), ((2, 3, 50), I8)),
    ("qbytes_softmax", lambda: (e(7, dtype=E4M3), e(), e()), ((7,), E4M3)),
]


@pytest.mark.parametrize("name,args,expected", CASES, ids=[f"{c[0]}-{i}" for i, c in enumerate(CASES)])
def test_fake_matches_cuda_allocation(name, args, expected):
    with FakeTensorMode():
        out = getattr(Q, name)(*args())
    shape, dtype = expected
    assert tuple(out.shape) == shape and out.dtype == dtype and out.device.type == "cuda"
    assert out.is_contiguous()


def test_every_defined_op_has_a_fake_and_a_case():
    with open(SOURCE) as f:
        names = re.findall(r'^_define\("(\w+)"', f.read(), flags=re.M)
    assert set(names) == set(library_attention.FAKE_IMPLS) == {c[0] for c in CASES}
    for name in names:
        assert torch._library.simple_registry.singleton.find("quanto::" + name).fake_impl.kernel is not None, name


def test_fake_checks_are_the_cuda_checks():
    with FakeTensorMode():
        with pytest.raises(ValueError, match="expects A"):
            Q.qbytes_bmm(e(4, 5, 64, dtype=I8), e(4, 63, 7, dtype=I8), e(), e())
        with pytest.raises(ValueError, match="per tensor"):
            Q.qbytes_bmm(e(4, 5, 64, dtype=I8), e(4, 64, 7, dtype=I8), e(2), e())
        with pytest.raises(NotImplementedError):
            Q.qbytes_softmax(e(4, 5), e(), e())


def test_bmm_oracle_exact_above_fp32_range():
    """K = 4096 of -128 * -128: sums reach 2^26, where an fp32 accumulation is no longer exact; the oracle's is."""
    a = np.full((1, 1, 4096), -128, np.int8)
    b = np.full((1, 4096, 1), -128, np.int8)
    b[0, 0, 0] = -127
    out = AO.qbytes_bmm(a, b, 1.0, 1.0, "f32")
    assert out[0, 0, 0] == np.float32(4096 * 16384 - 128)


def test_softmax_oracle_flags_midpoints():
    """A row of two equal codes: softmax 0.5 exactly, 0.5 / (1/127) = 63.5 is a rounding tie -> flagged."""
    codes, flags = AO.qbytes_softmax(np.array([[3, 3]], np.int8), "int8", 0.5, "f32")
    assert flags.all()
    codes, flags = AO.qbytes_softmax(np.array([[3]], np.int8), "int8", 0.5, "f32")
    assert codes[0, 0] == 127 and not flags.any()


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="fixture not generated")
def test_oracle_matches_reference_fixture():
    g = np.load(GOLDEN)
    for tag in ("f32", "f16", "bf16"):
        sa, sb = (AO.to_f32(AO.from_f32(np.float32(g[k]), tag), tag) for k in ("bmm_sa", "bmm_sb"))
        assert np.array_equal(AO.qbytes_bmm(g["bmm_a"], g["bmm_b"], sa, sb, tag), g[f"bmm_out_{tag}"]), tag
    for q_tag in ("int8", "e4m3fn", "e5m2", "e4m3fnuz"):
        for tag in ("f32", "bf16"):
            ref, flags = AO.qbytes_softmax(g[f"sm_in_{q_tag}"], q_tag, float(g["sm_scale"]), tag)
            got = g[f"sm_out_{q_tag}_{tag}"]
            diff = AO.code_distance(got, ref, q_tag)
            assert np.all(diff[~flags] == 0) and np.all(diff <= 1), (q_tag, tag)
            assert np.array_equal(AO.softmax_out_scale(q_tag, tag).reshape(-1), g[f"sm_scale_out_{q_tag}_{tag}"].reshape(-1))
