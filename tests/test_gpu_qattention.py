"""Quantized attention on the GPU: quanto::qbytes_bmm (every route) bit for bit against the exact oracle,
quanto::qbytes_softmax under its parity contract, the layout ops of the activation table, and an attention block of
frozen qint8 QLinears with qint8 activations, eager and under torch.compile."""
import math
import os

import numpy as np
import pytest
import torch

from helpers import ROOT, torch_to_bits
from oracle import attention_oracle as AO
from oracle import quanto_oracle as O

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

import quanto_b200 as q  # noqa: E402
from quanto_b200 import _native as N  # noqa: E402
from quanto_b200.tensor.activations import ActivationQBytesTensor, quantize_activation  # noqa: E402

DEV = torch.device("cuda:0")
DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
QDT = {"int8": torch.int8, "e4m3fn": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2, "e4m3fnuz": torch.float8_e4m3fnuz}
QTYPE = {"int8": q.qint8, "e4m3fn": q.qfloat8_e4m3fn, "e5m2": q.qfloat8_e5m2, "e4m3fnuz": q.qfloat8_e4m3fnuz}
GOLDEN = os.path.join(ROOT, "tests", "golden", "qattention.npz")


def exact_bmm(a, b, sa, sb):
    """The oracle's formula on the device: the int sum in float64 (exact below 2^53), then the reference's roundings."""
    acc = torch.bmm(a.double(), b.double()).float()
    s = (sa * sb).float()
    return (acc * s).to(sa.dtype)


def make_b(bt, k, n, layout, gen):
    """B [bt, K, N] int8 in one of the layouts attention produces: 'k' K-contiguous (a transposed key), 'n'
    N-contiguous (a value), 'x' one [K, N] matrix expanded over the batch (stride 0)."""
    if layout == "k":
        return torch.randint(-128, 128, (bt, n, k), dtype=torch.int8, device=DEV, generator=gen).transpose(1, 2)
    if layout == "n":
        return torch.randint(-128, 128, (bt, k, n), dtype=torch.int8, device=DEV, generator=gen)
    return torch.randint(-128, 128, (1, k, n), dtype=torch.int8, device=DEV, generator=gen).expand(bt, k, n)


# (batch, M, N, K, B layout, scale dtype, route); route None = automatic
BMM_CASES = [
    (1, 1, 1, 16, "k", "bf16", None),
    (1, 5, 5, 10, "n", "f32", None),
    (10, 64, 64, 64, "k", "f16", None),
    (10, 64, 200, 128, "n", "bf16", None),
    (10, 200, 64, 16, "x", "f32", None),
    (96, 200, 5, 64, "k", "bf16", None),
    (96, 5, 200, 128, "n", "f16", None),
    (32, 2048, 2048, 128, "k", "bf16", None),
    (32, 2048, 2048, 128, "n", "bf16", None),
    (1, 2048, 2048, 4096, "k", "bf16", None),
    (10, 200, 64, 1024, "n", "f32", None),
    (10, 64, 2048, 1024, "x", "bf16", None),
    (1, 2048, 1, 4096, "k", "f16", None),
    (10, 64, 200, 128, "k", "bf16", N.ROUTE_BMM_TRANSPOSE),
    (10, 200, 64, 64, "x", "f16", N.ROUTE_BMM_TRANSPOSE),
    (10, 64, 200, 128, "k", "bf16", N.ROUTE_BMM_SIMT),
    (10, 200, 5, 64, "n", "f32", N.ROUTE_BMM_SIMT),
    (96, 5, 64, 10, "x", "f16", N.ROUTE_BMM_SIMT),
    (1, 2048, 200, 4096, "n", "bf16", N.ROUTE_BMM_SIMT),
]


@pytest.mark.parametrize("bt,m,n,k,layout,tag,route", BMM_CASES)
def test_bmm_bit_exact(bt, m, n, k, layout, tag, route):
    gen = torch.Generator(device=DEV).manual_seed(bt * 7919 + m * 31 + n * 17 + k)
    a = torch.randint(-128, 128, (bt, m, k), dtype=torch.int8, device=DEV, generator=gen)
    b = make_b(bt, k, n, layout, gen)
    sa = (torch.rand((), device=DEV, generator=gen) / 100 + 1e-4).to(DT[tag])
    sb = (torch.rand((), device=DEV, generator=gen) / 100 + 1e-4).to(DT[tag])
    if route is None:
        out = torch.ops.quanto.qbytes_bmm(a, b, sa, sb)
    else:
        with N.test_override(N.OVR_BMM_ROUTE, route):
            out = torch.ops.quanto.qbytes_bmm(a, b, sa, sb)
    family = N.load().qb200_last_kernel_family()
    tc = k % 16 == 0
    expected = {None: (1 if layout == "k" else 4) if tc else 2, N.ROUTE_BMM_TRANSPOSE: 4 if tc else 2,
                N.ROUTE_BMM_SIMT: 2}[route]
    assert family == expected
    assert out.shape == (bt, m, n) and out.dtype == DT[tag]
    ref = exact_bmm(a, b, sa, sb)
    assert torch.equal(out, ref), float((out.float() - ref.float()).abs().max())
    if k <= 1024:  # there the reference's fp32 bmm is exact: the same bits as the reference itself
        fp32 = (torch.bmm(a.float(), b.float()) * (sa * sb).float()).to(DT[tag])
        assert torch.equal(out, fp32)


@pytest.mark.parametrize("tile", [(64, 128), (64, 256), (128, 128), (128, 256)])
def test_bmm_every_tile(tile):
    gen = torch.Generator(device=DEV).manual_seed(5)
    a = torch.randint(-128, 128, (3, 200, 96), dtype=torch.int8, device=DEV, generator=gen)
    b = make_b(3, 96, 300, "k", gen)
    s = torch.tensor(0.01, dtype=torch.bfloat16, device=DEV)
    with N.test_override(N.OVR_TILE_M, tile[0]), N.test_override(N.OVR_QBYTES_TILE_N, tile[1]):
        out = torch.ops.quanto.qbytes_bmm(a, b, s, s)
    assert torch.equal(out, exact_bmm(a, b, s, s))


def test_bmm_numpy_oracle_and_golden():
    rng = np.random.default_rng(3)
    a = rng.integers(-128, 128, (2, 5, 10), dtype=np.int8)
    b = rng.integers(-128, 128, (2, 10, 6), dtype=np.int8)
    for tag in ("f32", "f16", "bf16"):
        sa, sb = O.to_f32(O.from_f32(np.float32(0.0123), tag), tag), O.to_f32(O.from_f32(np.float32(0.0456), tag), tag)
        out = torch.ops.quanto.qbytes_bmm(torch.from_numpy(a).to(DEV), torch.from_numpy(b).to(DEV),
                                          torch.tensor(float(sa), dtype=DT[tag], device=DEV),
                                          torch.tensor(float(sb), dtype=DT[tag], device=DEV))
        assert np.array_equal(torch_to_bits(out), AO.qbytes_bmm(a, b, sa, sb, tag))
    if os.path.exists(GOLDEN):
        g = np.load(GOLDEN)
        for tag in ("f32", "f16", "bf16"):
            out = torch.ops.quanto.qbytes_bmm(torch.from_numpy(g["bmm_a"]).to(DEV), torch.from_numpy(g["bmm_b"]).to(DEV),
                                              torch.tensor(float(g["bmm_sa"]), dtype=DT[tag], device=DEV),
                                              torch.tensor(float(g["bmm_sb"]), dtype=DT[tag], device=DEV))
            assert np.array_equal(torch_to_bits(out), g[f"bmm_out_{tag}"])


def random_codes(shape, q_tag, gen):
    if q_tag == "int8":
        return torch.randint(-127, 128, shape, dtype=torch.int8, device=DEV, generator=gen)
    # finite codes only: scale * payload of a calibrated activation
    x = torch.randn(shape, device=DEV, generator=gen) * (O.FP8_MAX[q_tag] / 4)
    return x.clamp(-O.FP8_MAX[q_tag], O.FP8_MAX[q_tag]).to(QDT[q_tag])


@pytest.mark.parametrize("cols", [1, 7, 2048, 40000])
@pytest.mark.parametrize("q_tag", ["int8", "e4m3fn", "e5m2", "e4m3fnuz"])
@pytest.mark.parametrize("tag", ["bf16", "f32"])
def test_softmax_contract(cols, q_tag, tag):
    gen = torch.Generator(device=DEV).manual_seed(cols + len(q_tag))
    rows = 24 if cols < 40000 else 6
    data = random_codes((rows, cols), q_tag, gen)
    scale = torch.tensor(0.05 if q_tag == "int8" else 0.05 / 32, dtype=DT[tag], device=DEV)
    out_scale = torch.tensor(1 / AO.QMAX[q_tag], dtype=DT[tag], device=DEV)
    out = torch.ops.quanto.qbytes_softmax(data, scale, out_scale)
    assert out.dtype == data.dtype and out.shape == data.shape
    codes = torch_to_bits(data.view(torch.uint8) if q_tag != "int8" else data)
    s32 = O.to_f32(torch_to_bits(scale), tag) if tag != "f32" else np.float32(scale.item())
    ref, flags = AO.qbytes_softmax(codes, q_tag, float(s32), tag)
    got = torch_to_bits(out.view(torch.uint8) if q_tag != "int8" else out)
    diff = AO.code_distance(got, ref, q_tag)
    assert np.all(diff[~flags] == 0), int(np.sum(diff[~flags] != 0))
    assert np.all(diff[flags] <= 1)


def test_softmax_table_entry_and_fallback():
    gen = torch.Generator(device=DEV).manual_seed(9)
    x = torch.randn(4, 3, 50, device=DEV, generator=gen, dtype=torch.bfloat16)
    qx = quantize_activation(x, qtype=q.qint8, scale=torch.tensor(0.02, dtype=torch.bfloat16, device=DEV))
    y = torch.softmax(qx, dim=-1)
    assert isinstance(y, ActivationQBytesTensor) and y.qtype == q.qint8
    out_scale = torch.tensor(1 / 127, dtype=torch.bfloat16, device=DEV)
    assert torch.equal(y._scale, out_scale)
    assert torch.equal(y._data, torch.ops.quanto.qbytes_softmax(qx._data, qx._scale, out_scale))
    # another dim: the reference's composition on the existing kernels
    z = torch.softmax(qx, dim=1)
    ref = quantize_activation(torch.softmax(qx.dequantize(), dim=1), qtype=q.qint8, scale=out_scale)
    assert isinstance(z, ActivationQBytesTensor) and torch.equal(z._data, ref._data)


def _layout_cases():
    return [
        ("view", lambda t: t.view(4, 30, 8)),
        ("transpose", lambda t: t.transpose(1, 2)),
        ("permute", lambda t: t.permute(2, 0, 1)),
        ("expand", lambda t: t[:, None].expand(4, 3, 6, 40)),
        ("select", lambda t: t[:, 2]),
        ("slice", lambda t: t[:, 1:5]),
        ("unsqueeze", lambda t: t.unsqueeze(1)),
        ("clone", lambda t: t.transpose(1, 2).clone()),
        ("contiguous", lambda t: t.transpose(1, 2).contiguous()),
        ("reshape", lambda t: t.transpose(1, 2).reshape(4, -1)),
        ("t", lambda t: t[0].t()),
        ("split", lambda t: t.split(2, dim=1)[1]),
        ("cat", lambda t: torch.cat([t, t], dim=1)),
        ("stack", lambda t: torch.stack([t, t], dim=0)),
        ("neg", lambda t: -t),
        ("relu", lambda t: torch.relu(t)),
    ]


@pytest.mark.parametrize("name,fn", _layout_cases(), ids=[c[0] for c in _layout_cases()])
def test_layout_ops_stay_quantized(name, fn):
    gen = torch.Generator(device=DEV).manual_seed(11)
    x = torch.randn(4, 6, 40, device=DEV, generator=gen, dtype=torch.bfloat16)
    qx = quantize_activation(x, qtype=q.qint8, scale=torch.tensor(0.03, dtype=torch.bfloat16, device=DEV))
    y = fn(qx)
    assert isinstance(y, ActivationQBytesTensor), type(y)
    ref = fn(qx.dequantize())
    assert y.shape == ref.shape
    assert torch.equal(y.dequantize(), ref)
    assert torch.equal(y._scale, qx._scale)


def test_scalar_div_mul_only_touch_the_scale():
    x = torch.randn(4, 6, 40, device=DEV, dtype=torch.bfloat16)
    s = torch.tensor(0.03, dtype=torch.bfloat16, device=DEV)
    qx = quantize_activation(x, qtype=q.qint8, scale=s)
    for y, scale in ((qx / 3.0, s / 3.0), (qx * 0.5, 0.5 * s), (2.0 * qx, 2.0 * s)):
        assert isinstance(y, ActivationQBytesTensor)
        assert y._data is qx._data and torch.equal(y._scale, scale)


def test_layout_strides_match_oracle():
    x = torch.randn(4, 6, 40, device=DEV, dtype=torch.bfloat16)
    qx = quantize_activation(x, qtype=q.qint8, scale=torch.tensor(0.03, dtype=torch.bfloat16, device=DEV))
    for op, args, y in [("transpose", (1, 2), qx.transpose(1, 2)), ("permute", ((2, 0, 1),), qx.permute(2, 0, 1)),
                        ("select", (1, 2), qx.select(1, 2))]:
        shape, strides = AO.layout_result(tuple(qx.shape), tuple(qx.stride()), op, *args)
        assert tuple(y.shape) == shape and tuple(y.stride()) == strides and y._data.stride() == strides


def test_float8_and_float_first_operand_dequantize():
    x = torch.randn(2, 8, 16, device=DEV, dtype=torch.bfloat16)
    s = torch.tensor(0.01, dtype=torch.bfloat16, device=DEV)
    a8 = quantize_activation(x, qtype=q.qfloat8_e4m3fn, scale=s)
    b8 = quantize_activation(x.transpose(1, 2).contiguous(), qtype=q.qfloat8_e4m3fn, scale=s)
    assert torch.equal(torch.bmm(a8, b8), torch.bmm(a8.dequantize(), b8.dequantize()))
    b = quantize_activation(x.transpose(1, 2).contiguous(), qtype=q.qint8, scale=s)
    assert torch.equal(torch.bmm(x, b), torch.bmm(x, b.dequantize()))


# ----------------------------------------------------------------------------------------------- attention block
class Attention(torch.nn.Module):
    """The attention block of the reference's tests/nn/test_qattention.py, with and without its rotary embedding."""

    def __init__(self, hidden=128, heads=4, rope=False):
        super().__init__()
        self.hidden, self.heads, self.head_dim, self.rope = hidden, heads, hidden // heads, rope
        self.q_proj = torch.nn.Linear(hidden, hidden, bias=False)
        self.k_proj = torch.nn.Linear(hidden, hidden, bias=False)
        self.v_proj = torch.nn.Linear(hidden, hidden, bias=False)
        self.o_proj = torch.nn.Linear(hidden, hidden, bias=False)
        inv_freq = 1.0 / (10000 ** (torch.arange(0, self.head_dim, 2).float() / self.head_dim))
        emb = torch.cat([torch.outer(torch.arange(1024).float(), inv_freq)] * 2, dim=-1)
        self.register_buffer("cos", emb.cos(), persistent=False)
        self.register_buffer("sin", emb.sin(), persistent=False)

    def forward(self, x):
        bsz, n, _ = x.shape
        qs = self.q_proj(x).view(bsz, n, self.heads, self.head_dim).transpose(1, 2)
        ks = self.k_proj(x).view(bsz, n, self.heads, self.head_dim).transpose(1, 2)
        vs = self.v_proj(x).view(bsz, n, self.heads, self.head_dim).transpose(1, 2)
        if self.rope:
            cos, sin = self.cos[:n].to(x.dtype), self.sin[:n].to(x.dtype)

            def rot(t):
                return torch.cat((-t[..., self.head_dim // 2:], t[..., : self.head_dim // 2]), dim=-1)

            qs, ks = qs * cos + rot(qs) * sin, ks * cos + rot(ks) * sin
        w = torch.matmul(qs, ks.transpose(2, 3)) / math.sqrt(self.head_dim)
        w = torch.nn.functional.softmax(w, dim=-1)
        out = torch.matmul(w, vs).transpose(1, 2).contiguous().reshape(bsz, n, self.hidden)
        return self.o_proj(out)


def quantized_block(rope, dtype=torch.float32):
    torch.manual_seed(0)
    att = Attention(rope=rope).to(dtype).to(DEV)
    x = torch.randn(10, 64, 128, device=DEV, dtype=dtype)
    outs = {}
    hooks = [getattr(att, n).register_forward_hook(lambda m, i, o, n=n: outs.__setitem__(n, (i[0], o)))
             for n in ("q_proj", "k_proj", "v_proj", "o_proj")]
    with torch.no_grad():
        att(x)
    for h in hooks:
        h.remove()
    for n in ("q_proj", "k_proj", "v_proj", "o_proj"):
        lin = getattr(att, n)
        ql = q.QLinear.from_module(lin, weights=q.qint8, activations=q.qint8)
        ql.freeze()
        ql = ql.to(DEV)
        ql.input_scale = q.absmax_scale(outs[n][0]).to(dtype)
        ql.output_scale = q.absmax_scale(outs[n][1]).to(dtype)
        setattr(att, n, ql)
    return att, x


@pytest.mark.parametrize("rope", [False, True], ids=["no-rope", "rope"])
def test_attention_block_matches_op_chain(rope):
    att, x = quantized_block(rope)
    seen = {}
    hooks = [getattr(att, n).register_forward_hook(lambda m, i, o, n=n: seen.__setitem__(n, o))
             for n in ("q_proj", "k_proj", "v_proj")]
    with torch.no_grad():
        y = att(x)
    for h in hooks:
        h.remove()
    qq, kk, vv = seen["q_proj"], seen["k_proj"], seen["v_proj"]
    for t in (qq, kk, vv):
        assert isinstance(t, ActivationQBytesTensor)
    bsz, n, H, D = 10, 64, att.heads, att.head_dim
    with torch.no_grad():
        def heads(t):
            return t._data.view(bsz, n, H, D).transpose(1, 2)

        if rope:  # the rotary products dequantize: the chain is the float attention of the dequantized projections
            def hd(t):
                return t.dequantize().view(bsz, n, H, D).transpose(1, 2)

            cos, sin = att.cos[:n], att.sin[:n]

            def rot(t):
                return torch.cat((-t[..., D // 2:], t[..., : D // 2]), dim=-1)

            qs, ks = hd(qq) * cos + rot(hd(qq)) * sin, hd(kk) * cos + rot(hd(kk)) * sin
            scores = torch.matmul(qs, ks.transpose(2, 3))
        else:  # q @ k^T: the exact int8 product
            scores = exact_bmm(heads(qq).reshape(-1, n, D), heads(kk).transpose(2, 3).reshape(-1, D, n), qq._scale,
                               kk._scale).view(bsz, H, n, n)
        w = torch.softmax(scores / math.sqrt(D), dim=-1)
        out = torch.matmul(w, vv.dequantize().view(bsz, n, H, D).transpose(1, 2))
        ref = att.o_proj(out.transpose(1, 2).contiguous().reshape(bsz, n, 128))
    assert torch.equal(y.dequantize() if isinstance(y, ActivationQBytesTensor) else y,
                       ref.dequantize() if isinstance(ref, ActivationQBytesTensor) else ref)


@pytest.mark.parametrize("rope", [False, True], ids=["no-rope", "rope"])
def test_attention_block_compiles_bit_exact(rope):
    att, x = quantized_block(rope)
    with torch.no_grad():
        eager = att(x)
        torch._dynamo.reset()
        compiled = torch.compile(att, backend="aot_eager")(x)

    def plain(t):
        return t.dequantize() if isinstance(t, ActivationQBytesTensor) else t

    assert torch.equal(plain(eager), plain(compiled))
