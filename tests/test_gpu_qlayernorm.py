"""quanto::qbytes_layer_norm and QLayerNorm on the GPU: the parity contract of oracle/layernorm_oracle.py over dtypes,
code types, input forms, affine forms and row lengths; parity with the ATen composition; the reference's golden
outputs; the module's routes; an encoder block eager, under torch.compile and in a CUDA graph."""
import math
import os
import zlib

import numpy as np
import pytest
import torch

from helpers import ROOT, torch_to_bits
from oracle import layernorm_oracle as LO
from oracle.quanto_oracle import to_f32

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

import quanto_b200 as q  # noqa: E402
from quanto_b200 import _native as N  # noqa: E402
from quanto_b200 import library_norm  # noqa: E402
from quanto_b200.tensor.activations import ActivationQBytesTensor, quantize_activation  # noqa: E402

DEV = torch.device("cuda:0")
DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
QDT = {"int8": torch.int8, "e4m3fn": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2, "e4m3fnuz": torch.float8_e4m3fnuz}
QTYPE = {"int8": q.qint8, "e4m3fn": q.qfloat8_e4m3fn, "e5m2": q.qfloat8_e5m2, "e4m3fnuz": q.qfloat8_e4m3fnuz}
QMAX = {"int8": 127.0, "e4m3fn": 448.0, "e5m2": 57344.0, "e4m3fnuz": 240.0}
GOLDEN = os.path.join(ROOT, "tests", "golden", "qlayernorm.npz")
HS = (1, 7, 32, 50, 768, 1024, 4096, 5120, 8192, 16384, 65536)


def family():
    return N.load().qb200_last_kernel_family()


def rows_for(h):
    return (1, 3, 4096) if h <= 50 else (1, 3, 1024) if h <= 1024 else (1, 3, 64) if h <= 8192 else (1, 3)


def make_input(rows, h, dt, gen):
    """Normal rows, a constant row, a row whose mean is large against its spread."""
    x = torch.randn(rows, h, generator=gen) * 2 + 0.5
    if rows >= 3:
        x[1] = 1.25
        x[2] = 24 + 0.05 * torch.randn(h, generator=gen)
    return x.to(dt)


def params(kind, h, dt, gen):
    w = (1 + 0.5 * torch.randn(h, generator=gen)).to(dt) if kind != "none" else None
    b = (0.5 * torch.randn(h, generator=gen)).to(dt) if kind == "affine" else None
    return w, b


def f32(t):
    return None if t is None else to_f32(torch_to_bits(t), {torch.float32: "f32", torch.float16: "f16",
                                                           torch.bfloat16: "bf16"}[t.dtype])


def ulp(v, tag):
    """The spacing of `tag` at the float32 values v."""
    v = np.abs(np.asarray(v, np.float32))
    if tag == "f16":
        return np.spacing(v.astype(np.float16)).astype(np.float64)
    sp = np.spacing(v).astype(np.float64)
    return sp * 2 ** 16 if tag == "bf16" else sp


def check_codes(codes, ref, flags, lo, hi, q_tag, what):
    dist = LO.code_distance(codes, ref, q_tag)
    bad = int(np.sum(dist[~flags] != 0))
    assert bad == 0, f"{what}: {bad} unflagged elements differ"
    ok = (dist <= 1) | LO.within_band(codes, lo, hi, q_tag)
    assert np.all(ok), f"{what}: flagged elements outside the contract (max {dist.max()} codes)"


@pytest.mark.parametrize("src", ["float", "int8", "e4m3fn", "e5m2", "e4m3fnuz"])
@pytest.mark.parametrize("out", ["int8", "e4m3fn", "e5m2", "e4m3fnuz", "float"])
@pytest.mark.parametrize("tag", ["f32", "f16", "bf16"])
def test_contract_sweep(tag, out, src):
    dt = DT[tag]
    gen = torch.Generator().manual_seed(zlib.crc32(f"{tag}{out}{src}".encode()))
    flagged = total = 0
    for i, h in enumerate(HS):
        for rows in rows_for(h):
            kind = ("affine", "weight", "none")[(i + rows) % 3]
            x = make_input(rows, h, dt, gen)
            w, b = params(kind, h, dt, gen)
            s_in = None
            if src != "float":
                s_in = torch.tensor(float(x.float().abs().max()) / QMAX[src], dtype=dt)
                xin = torch.ops.quanto.quantize_symmetric(x.to(DEV), QDT[src], None, s_in.to(DEV))
                xf = LO.dequantize(torch_to_bits(xin), src, f32(s_in), tag)
            else:
                xin = x.to(DEV)
                xf = f32(x)
            dev = [None if t is None else t.to(DEV) for t in (s_in, w, b)]
            what = f"{tag}/{src}->{out}/{kind}/rows={rows}/H={h}"
            if out == "float":
                y = torch.ops.quanto.qbytes_layer_norm(xin, dev[0], [h], dev[1], dev[2], 1e-5, None, None)
                assert family() == 6 and y.dtype == dt
                ref, flags = LO.layer_norm(xf, tag, f32(w), f32(b), 1e-5)
                y64, band = LO.affine(xf, f32(w), f32(b), 1e-5)
                got = f32(y)
                assert np.all(got[~flags] == ref[~flags]), f"{what}: unflagged floats differ"
                assert np.all(np.abs(got - y64) <= band + ulp(ref, tag)), f"{what}: outside the band"
                # one T ulp of rnd_T(y64) wherever the band is narrower than half an ulp; elsewhere (fp32 outputs,
                # y near zero after gamma * n + beta cancels, the constant rows) the band above bounds the error
                narrow = band < 0.5 * ulp(ref, tag)
                assert np.all((np.abs(got - ref) <= ulp(ref, tag))[narrow]), f"{what}: more than one ulp"
                continue
            else:
                # an fp32 scale with 16-bit data on the non-affine rows (a module before calibration), else T
                s_dt = torch.float32 if kind == "none" else dt
                y64, _ = LO.affine(xf, f32(w), f32(b), 1e-5)
                top = max(float(np.abs(y64[0]).max()), 0.1)  # y = 0 everywhere when H = 1 without a bias
                s_out = torch.tensor(top / (0.8 * QMAX[out]), dtype=s_dt)  # saturates the largest outputs
                codes = torch.ops.quanto.qbytes_layer_norm(xin, dev[0], [h], dev[1], dev[2], 1e-5, s_out.to(DEV),
                                                           QDT[out])
                assert family() == 6 and codes.dtype == QDT[out]
                ref, flags, lo, hi = LO.qlayer_norm(xf, tag, f32(w), f32(b), 1e-5, f32(s_out), out, band_codes=True)
                check_codes(torch_to_bits(codes), ref, flags, lo, hi, out, what)
            rand = np.ones(rows, bool)
            rand[1:3] = False  # the constant and the large-mean rows sit on boundaries by construction
            flagged += int(flags[rand].sum())
            total += int(flags[rand].size)
    frac = flagged / max(total, 1)
    print(f"{tag}/{src}->{out}: flagged {frac:.4%} of the random rows")
    assert frac < 0.01


@pytest.mark.parametrize("q_tag", list(QDT))
@pytest.mark.parametrize("tag", list(DT))
def test_composition_parity(tag, q_tag):
    """Within one code (or the band) of quantize_symmetric(F.layer_norm(...)) run by ATen on the GPU."""
    dt = DT[tag]
    gen = torch.Generator().manual_seed(7)
    for h, rows in ((32, 4096), (768, 512), (4096, 64), (16384, 8), (65536, 2)):
        x = make_input(rows, h, dt, gen).to(DEV)
        w, b = (t.to(DEV) for t in params("affine", h, dt, gen))
        s = torch.tensor(4.0 / QMAX[q_tag], dtype=dt, device=DEV)
        codes = torch.ops.quanto.qbytes_layer_norm(x, None, [h], w, b, 1e-5, s, QDT[q_tag])
        comp = torch.ops.quanto.quantize_symmetric(torch.nn.functional.layer_norm(x, [h], w, b, 1e-5), QDT[q_tag],
                                                   None, s)
        _, _, lo, hi = LO.qlayer_norm(f32(x), tag, f32(w), f32(b), 1e-5, f32(s), q_tag, band_codes=True)
        a, c = torch_to_bits(codes), torch_to_bits(comp)
        dist = LO.code_distance(a, c, q_tag)
        assert np.all((dist <= 1) | LO.within_band(a, lo, hi, q_tag)), f"{tag}/{q_tag}/H={h}: {dist.max()} codes"


def test_golden_through_the_op():
    g = np.load(GOLDEN)
    for i in range(int(g["cases"])):
        tag, q_tag, kind, src, h, eps = g[f"{i}_meta"]
        dt, h, eps = DT[str(tag)], int(h), float(eps)

        def dev(key, dtype):
            a = g[key]
            t = torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a.copy())
            return t.view(dtype).to(DEV)

        s_dt = torch.float32 if g[f"{i}_s"].dtype == np.float32 else dt
        s = dev(f"{i}_s", s_dt)
        w = dev(f"{i}_w", dt) if f"{i}_w" in g else None
        b = dev(f"{i}_b", dt) if f"{i}_b" in g else None
        if src == "codes":
            x = dev(f"{i}_x", QDT[str(q_tag)] if q_tag == "int8" else torch.uint8)
            if q_tag != "int8":
                x = x.view(QDT[str(q_tag)])
            s_in = dev(f"{i}_sin", dt)
            xf = LO.dequantize(g[f"{i}_x"], str(q_tag), to_f32(g[f"{i}_sin"], str(tag)), str(tag))
        else:
            x, s_in, xf = dev(f"{i}_x", dt), None, to_f32(g[f"{i}_x"], str(tag))
        codes = torch.ops.quanto.qbytes_layer_norm(x, s_in, [h], w, b, eps, s, QDT[str(q_tag)])
        s_tag = "f32" if s_dt == torch.float32 else str(tag)
        ref, flags, lo, hi = LO.qlayer_norm(xf, str(tag), None if w is None else f32(w), None if b is None else f32(b),
                                            eps, to_f32(g[f"{i}_s"], s_tag), str(q_tag), band_codes=True)
        check_codes(torch_to_bits(codes), ref, flags, lo, hi, str(q_tag), f"golden {i}")
        # the reference's own codes obey the same contract
        check_codes(g[f"{i}_out"], ref, flags, lo, hi, str(q_tag), f"golden ref {i}")


# --------------------------------------------------------------------------------------------------- module
def qnorm(h=768, dt=torch.bfloat16, qt=q.qint8, affine=True, bias=True):
    torch.manual_seed(0)
    norm = torch.nn.LayerNorm(h, elementwise_affine=affine, bias=bias).to(dt).to(DEV)
    with torch.no_grad():
        if norm.weight is not None:
            norm.weight.copy_(1 + 0.3 * torch.randn(h))
        if norm.bias is not None:
            norm.bias.copy_(0.3 * torch.randn(h))
    m = q.QLayerNorm.from_module(norm, activations=qt)
    m.output_scale = torch.tensor(5.0 / 127, dtype=m.output_scale.dtype, device=DEV)
    return norm, m


def count_quantizations(monkeypatch):
    calls = []
    orig = q.nn.quantize_activation

    def counting(*args, **kwargs):
        calls.append(1)
        return orig(*args, **kwargs)

    monkeypatch.setattr(q.nn, "quantize_activation", counting)
    return calls


@pytest.mark.parametrize("affine,bias", [(True, True), (True, False), (False, False)])
def test_module_routes_to_the_op(monkeypatch, affine, bias):
    norm, m = qnorm(affine=affine, bias=bias)
    calls = count_quantizations(monkeypatch)
    x = torch.randn(4, 9, 768, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        y = m(x)
        assert family() == 6
        op = torch.ops.quanto.qbytes_layer_norm(x, None, [768], m.weight, m.bias, m.eps, m.output_scale, torch.int8)
        xq = quantize_activation(x, qtype=q.qint8, scale=torch.tensor(0.05, dtype=torch.bfloat16, device=DEV))
        calls.clear()
        yq = m(xq)
        op_q = torch.ops.quanto.qbytes_layer_norm(xq._data, xq._scale, [768], m.weight, m.bias, m.eps, m.output_scale,
                                                  torch.int8)
    assert calls == []  # the output hook passed the op's codes through
    for out, ref in ((y, op), (yq, op_q)):
        assert isinstance(out, ActivationQBytesTensor) and out.qtype is q.qint8
        assert out._scale is m.output_scale and torch.equal(out._data, ref)
        assert out.dtype == m.output_scale.dtype  # float32 for a non-affine module, as the reference's


def test_module_disabled_hook_float_paths():
    norm, m = qnorm()
    m.disable_output_quantization()
    x = torch.randn(6, 768, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        y = m(x)
        assert torch.equal(y, norm(x))  # a float input: F.layer_norm, bit for bit
        xq = quantize_activation(x, qtype=q.qint8, scale=torch.tensor(0.05, dtype=torch.bfloat16, device=DEV))
        yq = m(xq)
        assert family() == 6
    ref = torch.ops.quanto.qbytes_layer_norm(xq._data, xq._scale, [768], m.weight, m.bias, m.eps, None, None)
    assert type(yq) is torch.Tensor and torch.equal(yq, ref)
    assert torch.allclose(yq.float(), norm(xq.dequantize()).float(), atol=0.05)


def test_module_state_dict_round_trip_and_to():
    _, m = qnorm(qt=q.qfloat8_e4m3fn)
    sd = m.state_dict()
    _, m2 = qnorm(qt=q.qfloat8_e4m3fn)
    m2.output_scale = torch.tensor(1.0, dtype=torch.bfloat16, device=DEV)
    m2.load_state_dict(sd)
    assert torch.equal(m2.output_scale, m.output_scale) and torch.equal(m2.weight, m.weight)
    x = torch.randn(5, 768, device=DEV, dtype=torch.bfloat16)
    with torch.no_grad():
        assert torch.equal(m(x)._data, m2(x)._data)
        cpu = m2.to("cpu")
        assert cpu.weight.device.type == "cpu" and cpu.output_scale.device.type == "cpu"
        back = cpu.to(DEV)
        assert torch.equal(back(x)._data, m(x)._data)


def test_module_training_takes_the_composition():
    norm, m = qnorm()
    x = torch.randn(4, 768, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    assert library_norm.qlayernorm_forward(m, x, ActivationQBytesTensor, True) is None
    y = m(x)
    assert isinstance(y, ActivationQBytesTensor)
    y.dequantize().float().sum().backward()
    assert x.grad is not None and m.weight.grad is not None and m.bias.grad is not None
    ref_x = x.detach().clone().requires_grad_(True)
    norm(ref_x).float().sum().backward()
    assert torch.allclose(x.grad.float(), ref_x.grad.float(), atol=1e-2)


# ---------------------------------------------------------------------------------------------- encoder block
class Encoder(torch.nn.Module):
    """Pre-LN encoder attention: LayerNorm -> q / k / v projections -> softmax(q k^T / sqrt(d)) v -> output projection."""

    def __init__(self, hidden=128, heads=4):
        super().__init__()
        self.hidden, self.heads, self.head_dim = hidden, heads, hidden // heads
        self.ln = torch.nn.LayerNorm(hidden)
        self.q_proj = torch.nn.Linear(hidden, hidden)
        self.k_proj = torch.nn.Linear(hidden, hidden)
        self.v_proj = torch.nn.Linear(hidden, hidden)
        self.o_proj = torch.nn.Linear(hidden, hidden)

    def forward(self, x):
        bsz, n, _ = x.shape
        h = self.ln(x)
        qs = self.q_proj(h).view(bsz, n, self.heads, self.head_dim).transpose(1, 2)
        ks = self.k_proj(h).view(bsz, n, self.heads, self.head_dim).transpose(1, 2)
        vs = self.v_proj(h).view(bsz, n, self.heads, self.head_dim).transpose(1, 2)
        w = torch.nn.functional.softmax(torch.matmul(qs, ks.transpose(2, 3)) / math.sqrt(self.head_dim), dim=-1)
        out = torch.matmul(w, vs).transpose(1, 2).contiguous().reshape(bsz, n, self.hidden)
        return self.o_proj(out)


def quantized_encoder(dtype=torch.float32):
    torch.manual_seed(0)
    enc = Encoder().to(dtype).to(DEV)
    x = torch.randn(8, 64, 128, device=DEV, dtype=dtype)
    outs = {}
    names = ("ln", "q_proj", "k_proj", "v_proj", "o_proj")
    hooks = [getattr(enc, n).register_forward_hook(lambda m, i, o, n=n: outs.__setitem__(n, (i[0], o))) for n in names]
    with torch.no_grad():
        enc(x)
    for h in hooks:
        h.remove()
    qn = q.QLayerNorm.from_module(enc.ln, activations=q.qint8)
    qn.output_scale = q.absmax_scale(outs["ln"][1]).to(dtype)
    enc.ln = qn
    for n in names[1:]:
        ql = q.QLinear.from_module(getattr(enc, n), weights=q.qint8, activations=q.qint8)
        ql.freeze()
        ql = ql.to(DEV)
        ql.input_scale = q.absmax_scale(outs[n][0]).to(dtype)
        ql.output_scale = q.absmax_scale(outs[n][1]).to(dtype)
        setattr(enc, n, ql)
    return enc, x


def plain(t):
    return t.dequantize() if isinstance(t, ActivationQBytesTensor) else t


def test_encoder_block_keeps_codes_and_matches_composition():
    enc, x = quantized_encoder()
    seen = {}
    h1 = enc.ln.register_forward_hook(lambda m, i, o: seen.__setitem__("ln", o))
    h2 = enc.q_proj.register_forward_pre_hook(lambda m, i: seen.__setitem__("q_in", i[0]))
    with torch.no_grad():
        y = enc(x)
    h1.remove()
    h2.remove()
    assert isinstance(seen["ln"], ActivationQBytesTensor) and seen["q_in"] is seen["ln"]
    # the composition: F.layer_norm, then quantize_symmetric, through the same projections and attention ops
    with torch.no_grad():
        ln = enc.ln
        hq = quantize_activation(torch.nn.functional.layer_norm(x, ln.normalized_shape, ln.weight, ln.bias, ln.eps),
                                 qtype=q.qint8, scale=ln.output_scale)
        dist = (hq._data.int() - seen["ln"]._data.int()).abs()
        assert int(dist.max()) <= 1 and float((dist != 0).float().mean()) < 0.01
        saved = enc.ln
        enc.ln = torch.nn.Identity()
        ref = enc(hq)
        enc.ln = saved
    err = (plain(y).float() - plain(ref).float()).abs().max()
    assert float(err) <= 0.05 * float(plain(ref).float().abs().max())


def test_encoder_block_compiles_and_graphs_equal_eager():
    enc, x = quantized_encoder()
    with torch.no_grad():
        eager = plain(enc(x))
        torch._dynamo.reset()
        c1 = plain(torch.compile(enc, backend="aot_eager", fullgraph=True)(x))
        torch._dynamo.reset()
        fn = torch.compile(enc, backend="cudagraphs", dynamic=False)
        fn(x)
        c2 = plain(fn(x)).clone()
    assert torch.equal(eager, c1)
    assert torch.equal(eager, c2)


def test_op_in_a_cuda_graph():
    h = 4096
    x = torch.randn(64, h, device=DEV, dtype=torch.bfloat16)
    w = torch.randn(h, device=DEV, dtype=torch.bfloat16)
    b = torch.randn(h, device=DEV, dtype=torch.bfloat16)
    s = torch.tensor(0.05, device=DEV, dtype=torch.bfloat16)
    eager = torch.ops.quanto.qbytes_layer_norm(x, None, [h], w, b, 1e-5, s, torch.float8_e4m3fn)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        torch.ops.quanto.qbytes_layer_norm(x, None, [h], w, b, 1e-5, s, torch.float8_e4m3fn)
    torch.cuda.current_stream().wait_stream(stream)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = torch.ops.quanto.qbytes_layer_norm(x, None, [h], w, b, 1e-5, s, torch.float8_e4m3fn)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.uint8), eager.view(torch.uint8))
    s.fill_(0.1)  # the scale is read on the device at every replay
    graph.replay()
    ref = torch.ops.quanto.qbytes_layer_norm(x, None, [h], w, b, 1e-5, s, torch.float8_e4m3fn)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.uint8), ref.view(torch.uint8))
