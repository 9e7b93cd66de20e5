"""CPU checks of the quantized layer norm: the float64 oracle against the reference's own outputs
(tests/golden/qlayernorm.npz) under the parity contract, the fake of quanto::qbytes_layer_norm for every input / output
form, every argument check, and QLayerNorm's construction and state dict against the reference's.

The contract's EPS = 1e-5 (oracle/layernorm_oracle.py) bounds the kernel's fp32 arithmetic, u = 2^-24:
  - the mean: each thread adds at most 32 cached values in order (128 for a 65536-element row), then at most 9 levels
    of a pairwise reduction: |error| <= (128 + 9) u sum|x| / H <= 137 u (|mu| + sigma) = 8.2e-6 sigma (1 + |mu| / sigma);
    a row of at most 16384 elements stays under 41 u = 2.4e-6 of the same;
  - the variance about that mean, the same sums: <= 139 u relative, so rstd = (var + eps)^-1/2 (correctly rounded) is
    off by <= 70 u = 4.2e-6 relative -- a |n| term;
  - x - mu, (x - mu) * rstd and the final gamma * n + beta: one rounding each, <= 3 u (|gamma| |n| + |beta|).
The sum stays under 1e-5 * (|gamma| (1 + |n| + |mu| / sigma) + |beta|).  torch's CPU kernel (x * rstd - mu * rstd with
float accumulation over at most 768 elements here) stays inside the same band, which the golden test checks.
"""
import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

import quanto_b200 as q
from oracle import layernorm_oracle as LO
from oracle.quanto_oracle import to_f32

import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "qlayernorm.npz")
BF16, F16, F32, I8 = torch.bfloat16, torch.float16, torch.float32, torch.int8
Q = torch.ops.quanto


def golden_cases():
    g = np.load(GOLDEN)
    for i in range(int(g["cases"])):
        tag, q_tag, kind, src, h, eps = g[f"{i}_meta"]
        x = g[f"{i}_x"]
        if src == "codes":
            xf = LO.dequantize(x, q_tag, to_f32(g[f"{i}_sin"], tag), tag)
        else:
            xf = to_f32(x, tag)
        w = to_f32(g[f"{i}_w"], tag) if f"{i}_w" in g else None
        b = to_f32(g[f"{i}_b"], tag) if f"{i}_b" in g else None
        s_tag = "f32" if g[f"{i}_s"].dtype == np.float32 else tag
        s = to_f32(g[f"{i}_s"], s_tag)
        yield dict(tag=tag, q_tag=q_tag, kind=kind, src=src, h=int(h), eps=float(eps), x=xf, w=w, b=b, s=s,
                   out=g[f"{i}_out"])


def check_contract(codes, ref, flags, lo, hi, q_tag, what):
    dist = LO.code_distance(codes, ref, q_tag)
    assert np.all(dist[~flags] == 0), f"{what}: {int(np.sum(dist[~flags] != 0))} unflagged elements differ"
    ok = (dist <= 1) | LO.within_band(codes, lo, hi, q_tag)
    assert np.all(ok), f"{what}: flagged elements outside the band (max {dist.max()} codes away)"
    print(f"{what}: flagged {float(np.mean(flags)):.4%}")


def test_oracle_matches_reference_golden():
    cases = list(golden_cases())
    assert len(cases) == 228
    assert {c["tag"] for c in cases} == {"f32", "f16", "bf16"}
    assert {c["q_tag"] for c in cases} == {"int8", "e4m3fn", "e5m2", "e4m3fnuz"}
    assert {c["kind"] for c in cases} == {"affine", "weight", "none"} and {c["src"] for c in cases} == {"float", "codes"}
    assert {c["h"] for c in cases} == {1, 32, 50, 768}
    flagged = total = 0
    for c in cases:
        ref, flags, lo, hi = LO.qlayer_norm(c["x"], c["tag"], c["w"], c["b"], c["eps"], c["s"], c["q_tag"],
                                            band_codes=True)
        what = f"{c['tag']}/{c['q_tag']}/{c['kind']}/{c['src']}/H={c['h']}"
        check_contract(c["out"], ref, flags, lo, hi, c["q_tag"], what)
        flagged += int(flags.sum())
        total += flags.size
    assert flagged / total < 0.01, f"flagged fraction {flagged / total:.4%}"


def test_golden_state_dict_keys_match():
    g = np.load(GOLDEN)
    for kind, (affine, bias) in {"affine": (True, True), "weight": (True, False), "none": (False, False)}.items():
        m = q.QLayerNorm.from_module(torch.nn.LayerNorm(32, elementwise_affine=affine, bias=bias), activations=q.qint8)
        sd = m.state_dict()
        assert list(sd.keys()) == list(g[f"sd_keys_{kind}"])
        assert [k for k, v in sd.items() if v is None] == [k for k in g[f"sd_none_{kind}"] if k]
        assert [str(v.dtype) for v in sd.values() if v is not None] == list(g[f"sd_dtypes_{kind}"])


def test_qcreate_and_construction():
    norm = torch.nn.LayerNorm(64).to(BF16)
    assert q.QLayerNorm.from_module(norm) is None
    assert q.QLayerNorm.from_module(norm, weights=q.qint8) is None
    m = q.QLayerNorm.from_module(norm, weights=q.qint8, activations=q.qfloat8_e4m3fn)
    assert m.weight_qtype is None and m.activation_qtype is q.qfloat8_e4m3fn
    assert m.weight.dtype == BF16 and m.output_scale.dtype == BF16 and not m.frozen
    assert torch.equal(m.weight, norm.weight) and torch.equal(m.bias, norm.bias)
    m.freeze()
    assert not m.frozen and m.weight.dtype == BF16  # the weights are never quantized
    plain = q.QLayerNorm.from_module(torch.nn.LayerNorm(64, elementwise_affine=False), activations=q.qint8)
    assert plain.weight is None and plain.bias is None and plain.output_scale.dtype == F32
    assert plain.output_scale.device.type == "cpu"  # from_module of a non-affine norm: the reference's CPU default


def e(*shape, dtype=BF16):
    return torch.empty(shape, dtype=dtype, device="cuda")


FORMS = [
    # (input, input_scale, weight, bias, output_scale, output_dtype) -> output dtype
    (lambda: (e(4, 8, 32), None, e(32), e(32), e(), I8), I8),
    (lambda: (e(4, 8, 32, dtype=F16), None, None, None, e(dtype=F32), torch.float8_e5m2), torch.float8_e5m2),
    (lambda: (e(5, 50, dtype=torch.float8_e4m3fn), e(), e(50), None, e(), torch.float8_e4m3fnuz),
     torch.float8_e4m3fnuz),
    (lambda: (e(5, 50, dtype=I8), e(dtype=F32), e(50, dtype=F32), e(50, dtype=F32), None, None), F32),
    (lambda: (e(2, 3, 4, 6, dtype=F32), None, None, None, None, None), F32),
]


@pytest.mark.parametrize("args,out_dtype", FORMS, ids=[str(i) for i in range(len(FORMS))])
def test_fake_shapes_and_dtypes(args, out_dtype):
    with FakeTensorMode():
        x, s_in, w, b, s_out, dt = args()
        shape = list(w.shape) if w is not None else [x.shape[-1]]
        out = Q.qbytes_layer_norm(x, s_in, shape, w, b, 1e-5, s_out, dt)
        assert tuple(out.shape) == tuple(x.shape) and out.dtype == out_dtype and out.device.type == "cuda"


BAD = [
    ("does not end", lambda: (e(4, 32), None, [16], None, None, None, None)),
    ("must be 8-bit codes", lambda: (e(4, 32), e(), [32], None, None, None, None)),
    ("one floating point element", lambda: (e(4, 32, dtype=I8), e(2), [32], None, None, None, None)),
    ("one floating point element", lambda: (e(4, 32, dtype=I8), e(dtype=I8), [32], None, None, None, None)),
    ("float32, float16 or bfloat16", lambda: (e(4, 32, dtype=I8), None, [32], None, None, None, None)),
    ("weight must be", lambda: (e(4, 32), None, [32], e(32, dtype=F16), None, None, None)),
    ("bias must be", lambda: (e(4, 32), None, [32], None, e(31), None, None)),
    ("not an 8-bit code dtype", lambda: (e(4, 32), None, [32], None, None, e(), BF16)),
    ("one float32 or", lambda: (e(4, 32), None, [32], None, None, e(2), I8)),
    ("one float32 or", lambda: (e(4, 32), None, [32], None, None, e(dtype=F16), I8)),
    ("needs an output scale", lambda: (e(4, 32), None, [32], None, None, None, I8)),
    ("is on cpu", lambda: (e(4, 32), None, [32], None, None, torch.ones((), dtype=BF16), I8)),
    ("is on cpu", lambda: (e(4, 32), None, [32], torch.ones(32, dtype=BF16), None, None, None)),
]


@pytest.mark.parametrize("match,args", BAD, ids=[str(i) for i in range(len(BAD))])
def test_every_check_raises(match, args):
    with FakeTensorMode(allow_non_fake_inputs=True):
        x, s_in, shape, w, b, s_out, dt = args()
        with pytest.raises(ValueError, match=match):
            Q.qbytes_layer_norm(x, s_in, shape, w, b, 1e-5, s_out, dt)


def test_fake_is_registered():
    from quanto_b200 import library_norm
    assert set(library_norm.FAKE_IMPLS) == {"qbytes_layer_norm"}
    assert torch._library.simple_registry.singleton.find("quanto::qbytes_layer_norm").fake_impl.kernel is not None
