"""Frozen QLinear models under torch.compile on the H100: compiled results equal eager bit for bit.

The compiled graphs call the same sm_90a kernels as eager code (the ops are opaque to the compiler), so every
comparison is `torch.equal`.
"""
import pytest
import torch
from torch._dynamo.testing import CompileCounterWithBackend

import quanto_b200 as q
from quanto_b200 import _native
from quanto_b200.tensor import PackedTensor, WeightQBitsTensor
from quanto_b200.tensor.function import NATIVE_GRAD_INPUT_MAX_M

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF16 = torch.bfloat16
MS = (1, 8, 12, 33, 300, 4096)
N, K = 512, 256  # per-axis weights are single 256-wide groups


def compile_fullgraph(model, backend):
    """torch's "cudagraphs" backend records one graph per compiled shape, so it is compiled static (one graph per M)."""
    return torch.compile(model, backend=backend, fullgraph=True, dynamic=False if backend == "cudagraphs" else None)

# (name, qtype, group size (None = per-axis), integer zero-point)
QBITS = [
    ("qint4-g128-shift", q.qint4, 128, False),
    ("qint4-g128-zp", q.qint4, 128, True),
    ("qint4-axis-shift", q.qint4, None, False),
    ("qint2-g64-zp", q.qint2, 64, True),
    ("qint2-axis-shift", q.qint2, None, False),
]
QBYTES = [("qint8", q.qint8), ("qfloat8_e4m3fn", q.qfloat8_e4m3fn), ("qfloat8_e5m2", q.qfloat8_e5m2),
          ("qfloat8_e4m3fnuz", q.qfloat8_e4m3fnuz)]
WEIGHTS = [w[0] for w in QBITS] + [w[0] for w in QBYTES]


@pytest.fixture(autouse=True)
def _fresh_dynamo():
    torch._dynamo.reset()
    torch._dynamo.utils.counters.clear()
    yield
    torch._dynamo.reset()


def qbits_linear(qtype, group, zeropoint, n=N, k=K, bias=True, seed=0):
    """A frozen QLinear whose packed weight comes from the on-device MaxOptimizer freeze (float shift or zero-point)."""
    torch.manual_seed(seed)
    lin = q.QLinear(k, n, bias=bias, dtype=BF16, device=DEV, weights=qtype)
    w = torch.randn(n, k, dtype=BF16, device=DEV) * 0.05
    g = group or k
    packed, scale, shift = torch.ops.quanto.quantize_qbits_max(w, qtype.bits, g, zeropoint)
    data = PackedTensor(packed, qtype.bits, torch.Size([n * k // g, g]), (g, 1))
    qw = WeightQBitsTensor(qtype, 0, group, w.size(), w.stride(), data, scale, shift)
    lin.weight = torch.nn.Parameter(qw, requires_grad=False)
    if bias:
        with torch.no_grad():
            lin.bias.copy_(torch.randn(n, dtype=BF16, device=DEV) * 0.1)
    return lin


def qbytes_linear(qtype, n=N, k=K, bias=True, activations=None, seed=0):
    torch.manual_seed(seed)
    base = torch.nn.Linear(k, n, bias=bias, dtype=BF16, device=DEV)
    with torch.no_grad():
        base.weight.mul_(4.0)
    lin = q.QLinear.from_module(base, weights=qtype, activations=activations)
    lin.freeze()
    return lin


def make_linear(name, bias=True):
    for wname, qtype, group, zp in QBITS:
        if wname == name:
            return qbits_linear(qtype, group, zp, bias=bias)
    return qbytes_linear(dict(QBYTES)[name], bias=bias)


def inputs(m, k=K, seed=1):
    torch.manual_seed(seed)
    return torch.randn(m, k, dtype=BF16, device=DEV)


@pytest.mark.parametrize("backend", ["aot_eager", "cudagraphs"])
@pytest.mark.parametrize("bias", [True, False], ids=["bias", "nobias"])
@pytest.mark.parametrize("weights", WEIGHTS)
def test_compiled_forward_equals_eager(weights, bias, backend):
    lin = make_linear(weights, bias)
    compiled = compile_fullgraph(lin, backend)
    with torch.no_grad():
        for m in MS:
            x = inputs(m)
            ref = lin(x)
            for _ in range(3):  # cudagraphs: warm-up, record, replay
                out = compiled(x).clone()
                assert torch.equal(out, ref), (weights, m)


def test_compiled_3d_activations_equal_eager():
    lin = make_linear("qint4-g128-shift")
    compiled = torch.compile(lin, backend="aot_eager", fullgraph=True)
    with torch.no_grad():
        x = inputs(2 * 33).reshape(2, 33, K)
        assert torch.equal(compiled(x), lin(x))


@pytest.mark.parametrize("weights", ["qint4-g128-shift", "qint8"])
def test_dynamic_token_count_compiles_once(weights):
    lin = make_linear(weights)
    counter = CompileCounterWithBackend("aot_eager")
    compiled = torch.compile(lin, backend=counter, fullgraph=True)
    with torch.no_grad():
        for m in (9, 17, 64, 300, 1000):
            x = inputs(m)
            torch._dynamo.mark_dynamic(x, 0)
            assert torch.equal(compiled(x), lin(x)), m
    assert counter.frame_count == 1


def test_dynamic_token_count_backward_compiles_once_per_route():
    """The input gradient picks its route on M in Python: one guard, one graph per route range, never a changed route."""
    lin = make_linear("qint4-g128-shift")
    counter = CompileCounterWithBackend("aot_eager")
    compiled = torch.compile(lin, backend=counter, fullgraph=True)
    for m in (16, 40, NATIVE_GRAD_INPUT_MAX_M, 200, 300):
        x = inputs(m).requires_grad_(True)
        torch._dynamo.mark_dynamic(x, 0)
        compiled(x).float().sum().backward()
        x_ref = x.detach().clone().requires_grad_(True)
        lin(x_ref).float().sum().backward()
        assert torch.equal(x.grad, x_ref.grad), m
    assert counter.frame_count <= 2


@pytest.mark.parametrize("backend", ["aot_eager", "cudagraphs"])
@pytest.mark.parametrize("m", [16, 300])
@pytest.mark.parametrize("weights", ["qint4-g128-shift", "qint4-g128-zp", "qint2-g64-zp", "qint8", "qfloat8_e4m3fn"])
def test_compiled_input_gradient_equals_eager(weights, m, backend):
    lin = make_linear(weights)
    compiled = compile_fullgraph(lin, backend)
    gO = torch.randn(m, N, dtype=BF16, device=DEV)
    x_ref = inputs(m).requires_grad_(True)
    lin(x_ref).backward(gO)
    for _ in range(3):
        x = inputs(m).requires_grad_(True)
        compiled(x).backward(gO)
        assert torch.equal(x.grad, x_ref.grad)


def _stream_k_decode_linear():
    """A decode-shaped qint4 linear whose M = 1 call runs the stream-K gemv (the route that needs the workspace)."""
    n, k = 4096, 4096
    lib = _native.load()
    assert lib.qb200_qbits_mm_workspace_bytes(1, n, k) > 0
    return qbits_linear(q.qint4, 128, False, n=n, k=k, bias=False, seed=3), k


def test_cudagraphs_replay_after_second_graph_in_pool():
    """A graph recorded while the stream-K workspace was first needed still replays correctly after a second graph was
    recorded in the same cudagraph-tree pool."""
    lin_a, k = _stream_k_decode_linear()
    lin_b = qbits_linear(q.qint4, 128, False, n=6144, k=k, bias=False, seed=4)
    fa = compile_fullgraph(lin_a, "cudagraphs")
    fb = compile_fullgraph(lin_b, "cudagraphs")
    with torch.no_grad():
        x1 = inputs(1, k)
        ref_a = lin_a(x1)
        for _ in range(3):
            assert torch.equal(fa(x1).clone(), ref_a)
        for m in (1, 8, 32):
            xb = inputs(m, k, seed=m)
            ref_b = lin_b(xb)
            for _ in range(3):
                assert torch.equal(fb(xb).clone(), ref_b), m
        for _ in range(5):
            assert torch.equal(fa(x1).clone(), ref_a)
            assert torch.equal(fb(inputs(8, k, seed=8)).clone(), lin_b(inputs(8, k, seed=8)))
    torch.cuda.synchronize()


def test_capture_uses_workspace_prepared_outside_it():
    """A hand-captured graph takes the device's capture workspace prepared by the eager warm-up; it allocates none."""
    lin, k = _stream_k_decode_linear()
    x = inputs(1, k)
    with torch.no_grad():
        ref = lin(x)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            lin(x)
        torch.cuda.current_stream().wait_stream(side)
        before = {key: t.data_ptr() for key, t in _native._workspaces.items()}
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = lin(x)
        assert {key: t.data_ptr() for key, t in _native._workspaces.items()} == before
        for _ in range(3):
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(out, ref)


@pytest.mark.parametrize("backend", ["aot_eager", "cudagraphs"])
@pytest.mark.parametrize("act", [q.qint8, q.qfloat8], ids=["qint8", "qfloat8"])
@pytest.mark.parametrize("first", ["qint8", "qint4"])
def test_quantized_activations_equal_eager(first, act, backend):
    """Input pre-hook, fused quantized-output linear and ActivationQBytesTensor outputs, as one graph."""
    torch.manual_seed(0)
    if first == "qint4":
        l1 = q.QLinear.from_module(torch.nn.Linear(K, N, dtype=BF16, device=DEV), weights=q.qint4, activations=act)
        l1.freeze()
    else:
        l1 = qbytes_linear(q.qint8, activations=act)
    l2 = qbytes_linear(act if act.dtype != torch.int8 else q.qint8, n=256, k=N, activations=act, seed=5)
    for lin in (l1, l2):
        lin.input_scale.fill_(0.02)
        lin.output_scale.fill_(0.05)
    model = torch.nn.Sequential(l1, l2)
    compiled = compile_fullgraph(model, backend)
    with torch.no_grad():
        for m in (1, 33, 300):
            x = inputs(m)
            ref = model(x)
            for _ in range(3):
                out = compiled(x)
                assert type(out) is type(ref)
                assert torch.equal(out._data.view(torch.uint8), ref._data.view(torch.uint8)), m
                assert torch.equal(out._scale, ref._scale)
    assert not torch._dynamo.utils.counters["graph_break"]


def test_two_layer_mlp_is_one_graph():
    up = qbits_linear(q.qint4, 128, False, n=2048, k=K, bias=False, seed=6)
    down = qbits_linear(q.qint4, 128, True, n=K, k=2048, bias=True, seed=7)
    model = torch.nn.Sequential(up, torch.nn.SiLU(), down)
    counter = CompileCounterWithBackend("aot_eager")
    compiled = torch.compile(model, backend=counter, fullgraph=True)
    with torch.no_grad():
        x = inputs(12)
        assert torch.equal(compiled(x), model(x))
    assert counter.frame_count == 1
    assert not torch._dynamo.utils.counters["graph_break"]
