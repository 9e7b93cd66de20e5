"""quanto::absmax_update_ and Calibration on the GPU: the reference's scale bits (tests/golden/calibration.npz) through
the op, edge sizes and alignments against the numpy oracle, one launch per update; calibrated modules bit-equal to the
ATen composition; the reference's streamline decisions and output qtypes; no host synchronisation; a calibration step
captured in a CUDA graph; quantize -> calibrate -> freeze -> state_dict -> requantize."""
import os

import numpy as np
import pytest
import torch

from helpers import ROOT
from oracle import calibration_oracle as CO

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

import quanto_b200 as q  # noqa: E402
from quanto_b200 import calibrate  # noqa: E402
from quanto_b200.tensor.activations import quantize_activation  # noqa: E402

DEV = torch.device("cuda:0")
GOLDEN = os.path.join(ROOT, "tests", "golden", "calibration.npz")
DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
ACTS = [q.qint8, q.qfloat8_e4m3fn, q.qfloat8_e5m2, q.qfloat8_e4m3fnuz]
BF16 = torch.bfloat16


def to_device(bits, tag):
    """T bit patterns -> a CUDA tensor of T."""
    if tag == "f32":
        return torch.from_numpy(np.asarray(bits, np.uint32).view(np.int32).copy()).view(torch.float32).to(DEV)
    return torch.from_numpy(np.asarray(bits, np.uint16).view(np.int16).copy()).view(DT[tag]).to(DEV)


def bits_of(t, tag):
    t = t.detach().reshape(-1).cpu()
    if tag == "f32":
        return t.view(torch.int32).numpy().view(np.uint32)
    return t.view(torch.int16).numpy().view(np.uint16)


def same(got, want, tag):
    """Equal bit patterns, or both NaN."""
    return got == want or (np.isnan(CO.values(np.array([got]), tag)[0]) and np.isnan(CO.values(np.array([want]), tag)[0]))


# ---------------------------------------------------------------------------------------------- the op, bit for bit
def test_op_reproduces_every_golden_scale():
    g = np.load(GOLDEN)
    n = sum(1 for k in g.files if k.endswith("_meta"))
    for c in range(n):
        code, qmax, momentum, count = g[f"{c}_meta"]
        tag = CO.TAGS[int(code)]
        s = g[f"{c}_s"]
        scale = to_device(s[:1], tag).reshape(())
        ptr = scale.data_ptr()
        for j in range(int(count)):
            torch.ops.quanto.absmax_update_(scale, to_device(g[f"{c}_x{j}"], tag), float(qmax), float(momentum))
            got = bits_of(scale, tag)[0]
            assert same(got, s[j + 1], tag), (c, j, tag, qmax, momentum, hex(got), hex(s[j + 1]))
        assert scale.data_ptr() == ptr


@pytest.mark.parametrize("tag", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("n, offset", [(1, 0), (1, 1), (7, 0), (7, 3), (8, 1), (4097, 0), (4097, 5), (1 << 20, 1),
                                       ((1 << 26) + 3, 0), ((1 << 26) + 3, 1)])
def test_op_sizes_and_alignments_match_the_oracle(tag, n, offset):
    """numel of 1, odd sizes, bases off the 16-byte boundary (scalar path) and 64M-element multi-CTA reductions, with
    the maximum placed in the scalar tail or deep inside; first-batch and momentum updates."""
    gen = torch.Generator(device=DEV).manual_seed(n + offset)
    buf = torch.randn(n + offset, generator=gen, device=DEV).to(DT[tag])
    x = buf[offset:]
    x[(n * 7) // 11] = -37.5  # a maximum far from the first element
    for qmax, momentum, start in ((127.0, 0.9, 1.0), (448.0, 0.37, 0.021), (57344.0, 0.99, 3.5e-4)):
        scale = torch.full((), start, dtype=DT[tag], device=DEV)
        start_v = CO.values(bits_of(scale, tag), tag)[0]
        torch.ops.quanto.absmax_update_(scale, x, qmax, momentum)
        want = CO.absmax_update(start_v, CO.values(bits_of(x, tag), tag), qmax, momentum, tag)
        assert bits_of(scale, tag)[0] == CO.bits_of(np.array([want], np.float32), tag)[0], (qmax, momentum)
    x[n - 1] = float("nan")  # a NaN in the last element (the scalar tail when unaligned) poisons the scale
    torch.ops.quanto.absmax_update_(scale, x, 127.0, 0.9)
    assert torch.isnan(scale)


def test_op_is_one_kernel_launch():
    x = torch.randn(1 << 22, device=DEV, dtype=BF16)
    scale = torch.ones((), device=DEV, dtype=BF16)
    torch.ops.quanto.absmax_update_(scale, x, 127.0, 0.9)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        torch.ops.quanto.absmax_update_(scale, x, 127.0, 0.9)
        torch.cuda.synchronize()
    kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and "memset" not in e.name.lower()]
    assert len(kernels) == 1 and "absmax_update_kernel" in kernels[0], kernels


def test_op_rejects_bad_arguments():
    x = torch.randn(16, device=DEV, dtype=BF16)
    for scale, base, qmax in ((torch.ones((), device=DEV), x, 127.0),
                              (torch.ones((), device=DEV, dtype=BF16), x[:0], 127.0),
                              (torch.ones(2, device=DEV, dtype=BF16), x, 127.0),
                              (torch.ones((), device=DEV, dtype=BF16), x, -1.0)):
        with pytest.raises(ValueError):
            torch.ops.quanto.absmax_update_(scale, base, qmax, 0.9)


# -------------------------------------------------------------------------------------------------------- modules
class Composition:
    """Run the Calibration mode on the ATen composition of the reference's formula."""

    def __enter__(self):
        calibrate._FORCE_COMPOSITION = True

    def __exit__(self, *exc):
        calibrate._FORCE_COMPOSITION = False


class MLP3(torch.nn.Module):
    def __init__(self, d=64):
        super().__init__()
        self.l1 = torch.nn.Linear(d, 128)
        self.l2 = torch.nn.Linear(128, 128)
        self.l3 = torch.nn.Linear(128, d)

    def forward(self, x):
        return self.l3(torch.nn.functional.silu(self.l2(self.l1(x))))


class Encoder(torch.nn.Module):
    """The pre-LN block of oracle/gen_golden_calibration.py."""

    def __init__(self, d=64):
        super().__init__()
        self.ln1 = torch.nn.LayerNorm(d)
        self.q = torch.nn.Linear(d, d)
        self.k = torch.nn.Linear(d, d)
        self.v = torch.nn.Linear(d, d)
        self.o = torch.nn.Linear(d, d)
        self.ln2 = torch.nn.LayerNorm(d)
        self.fc1 = torch.nn.Linear(d, 4 * d)
        self.fc2 = torch.nn.Linear(4 * d, d)

    def forward(self, x):
        h = self.ln1(x)
        a = torch.softmax(torch.bmm(self.q(h), self.k(h).transpose(1, 2)), dim=-1)
        x = x + self.o(torch.bmm(a, self.v(h)))
        return x + self.fc2(torch.nn.functional.gelu(self.fc1(self.ln2(x))))


def frozen_encoder():
    torch.manual_seed(0)
    model = Encoder().to(DEV, BF16)
    q.quantize(model, weights=q.qint8, activations=q.qint8)
    q.freeze(model)
    return model


def scales(model):
    return {n: (m.input_scale.clone(), m.output_scale.clone()) for n, m in model.named_modules()
            if isinstance(m, q.QModuleMixin)}


def calibrate_both(make, batches, **kw):
    """Calibrate two models built by `make`, natively and on the composition; return both."""
    native, comp = make(), make()
    with torch.no_grad():
        for x in batches:
            with q.Calibration(**kw):
                native(x)
            with Composition(), q.Calibration(**kw):
                comp(x)
    return native, comp


def raw(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def assert_same_scales(a, b):
    sa, sb = scales(a), scales(b)
    assert sa.keys() == sb.keys()
    for n in sa:
        for x, y in zip(sa[n], sb[n]):
            assert x.dtype == y.dtype and x.shape == y.shape and torch.equal(raw(x), raw(y)), (n, x, y)
        assert not torch.all(sa[n][1] == 1), n


def batches(shape, k=4, dtype=BF16, seed=0):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.randn(shape, generator=gen, device=DEV).to(dtype) * (0.5 + i) for i in range(k)]


@pytest.mark.parametrize("weights", [q.qint4, q.qint8, q.qfloat8_e4m3fn])
@pytest.mark.parametrize("frozen", [False, True])
def test_qlinear_scales_equal_the_composition(weights, frozen):
    def make():
        torch.manual_seed(0)
        m = q.QLinear.from_module(torch.nn.Linear(256, 384).to(DEV, BF16), weights=weights, activations=q.qint8)
        if frozen:
            m.freeze()
        return m

    native, comp = calibrate_both(make, batches((3, 17, 256)), momentum=0.7)
    assert_same_scales(native, comp)
    buf = native.input_scale
    with torch.no_grad(), q.Calibration():
        native(batches((3, 17, 256), k=1, seed=5)[0])
    assert native.input_scale is buf  # updated in place


def test_qconv2d_and_qlayernorm_scales_equal_the_composition():
    def conv():
        torch.manual_seed(0)
        return q.QConv2d.from_module(torch.nn.Conv2d(8, 16, 3, padding=1).to(DEV, BF16), weights=q.qint8,
                                     activations=q.qint8)

    native, comp = calibrate_both(conv, batches((2, 8, 12, 12)))
    assert_same_scales(native, comp)
    for affine in (True, False):
        def ln():
            torch.manual_seed(0)
            return q.QLayerNorm.from_module(torch.nn.LayerNorm(320, elementwise_affine=affine).to(DEV, BF16),
                                            activations=q.qint8)

        native, comp = calibrate_both(ln, batches((4, 9, 320)), momentum=0.5)
        # a non-affine QLayerNorm keeps float32 scales; the bf16 activation then takes the composition, which promotes
        assert_same_scales(native, comp)


@pytest.mark.parametrize("streamline", [True, False])
def test_encoder_scales_equal_the_composition(streamline):
    native, comp = calibrate_both(frozen_encoder, batches((2, 16, 64)), streamline=streamline)
    assert_same_scales(native, comp)


# ---------------------------------------------------------------------------------------- streamline and qtypes
@pytest.mark.parametrize("tag, cls, shape", [("mlp3", MLP3, (4, 64)), ("encoder", Encoder, (2, 8, 64))])
@pytest.mark.parametrize("streamline", [True, False])
def test_streamline_decisions_equal_the_reference(tag, cls, shape, streamline):
    g = np.load(GOLDEN)
    torch.manual_seed(1)
    model = cls().to(DEV, BF16)
    q.quantize(model, weights=q.qint8, activations=q.qint8)
    with torch.no_grad(), q.Calibration(streamline=streamline):
        model(torch.randn(shape, device=DEV, dtype=BF16))
    qmods = [(n, m) for n, m in model.named_modules() if isinstance(m, q.QModuleMixin)]
    assert [n for n, _ in qmods] == [str(n) for n in g[f"{tag}_names"]]
    assert [("output" in m._quantize_hooks) for _, m in qmods] == list(g[f"{tag}_{int(streamline)}_live"])


def random_qactivation(shape, qtype, seed=0):
    x = torch.randn(shape, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV).to(BF16)
    return quantize_activation(x, qtype=qtype, scale=calibrate.absmax_scale(x, qtype))


@pytest.mark.parametrize("activations", ACTS, ids=lambda t: t.name)
@pytest.mark.parametrize("batch_size, tokens, embeddings", [(1, 32, 32), (10, 10, 32)])
@pytest.mark.parametrize("use_bias", [True, False])
def test_calibrate_qlinear_output_qtype(activations, batch_size, tokens, embeddings, use_bias):
    """tests/nn/test_calibrate.py of the reference, on the GPU in bf16."""
    linear = torch.nn.Linear(embeddings, embeddings, bias=use_bias).to(DEV, BF16)
    qlinear = q.QLinear.from_module(linear, weights=q.qint8, activations=activations)
    qinputs = random_qactivation((batch_size, tokens, embeddings), activations)
    with torch.no_grad():
        qlinear(qinputs)
    assert torch.all(qlinear.input_scale == 1) and torch.all(qlinear.output_scale == 1)
    with torch.no_grad(), q.Calibration():
        qout = qlinear(qinputs)
    assert qout.qtype == activations
    assert torch.any(qlinear.input_scale != 1) and torch.any(qlinear.output_scale != 1)


@pytest.mark.parametrize("activations", ACTS, ids=lambda t: t.name)
def test_calibrate_chained_qlinears_output_qtype(activations):
    """Two chained QLinears inside a parent module: both calibrate, and the output keeps the activation qtype."""
    model = torch.nn.Sequential(torch.nn.Linear(32, 48), torch.nn.Linear(48, 32)).to(DEV, BF16)
    q.quantize(model, weights=q.qint8, activations=activations)
    with torch.no_grad(), q.Calibration():
        qout = model(random_qactivation((1, 10, 32), activations))
    for m in model:
        assert torch.any(m.input_scale != 1) and torch.any(m.output_scale != 1)
    assert qout.qtype == activations


def test_input_scale_uses_momentum_0_9_whatever_the_mode_says():
    """The reference's input hook never receives the mode's momentum: pinned against the numpy oracle."""
    m = q.QLinear.from_module(torch.nn.Linear(64, 64).to(DEV, BF16), weights=q.qint8, activations=q.qint8)
    xs = batches((4, 64), k=3, seed=9)
    want = np.float32(1.0)
    for x in xs:
        with torch.no_grad(), q.Calibration(momentum=0.5):
            m(x)
        want = CO.absmax_update(want, CO.values(bits_of(x, "bf16"), "bf16"), 127.0, 0.9, "bf16")
    assert bits_of(m.input_scale, "bf16")[0] == CO.bits_of(np.array([want], np.float32), "bf16")[0]
    with_half = np.float32(1.0)
    for x in xs:
        with_half = CO.absmax_update(with_half, CO.values(bits_of(x, "bf16"), "bf16"), 127.0, 0.5, "bf16")
    assert with_half != want  # the batches tell the two momenta apart


class SharedTwice(torch.nn.Module):
    """One module applied to two inputs; its first output is consumed after the second call."""

    def __init__(self, d=64):
        super().__init__()
        self.shared = torch.nn.Linear(d, d)
        self.head = torch.nn.Linear(d, d)

    def forward(self, x):
        first = self.shared(x)
        self.shared(x * 4)
        return self.head(first)


def test_outputs_keep_their_scale_after_later_updates():
    """The in-place update must not reach outputs already handed out: the reference rebinds the buffer, so an earlier
    output keeps the scale it was quantized with (a module applied twice, an output kept across batches)."""
    def make():
        torch.manual_seed(0)
        model = SharedTwice().to(DEV, BF16)
        q.quantize(model, weights=q.qint8, activations=q.qint8)
        return model

    native, comp = calibrate_both(make, batches((8, 64), k=3, seed=4), streamline=False, momentum=0.5)
    assert_same_scales(native, comp)
    kept = []
    with torch.no_grad():
        for x in batches((8, 64), k=2, seed=6):
            with q.Calibration(streamline=False):
                kept.append(native.shared(x))
    assert isinstance(kept[0], q.ActivationQBytesTensor)
    assert not torch.equal(kept[0]._scale, native.shared.output_scale)
    assert torch.equal(kept[1]._scale, native.shared.output_scale)


# ------------------------------------------------------------------------------------ no sync, graphs, round trip
def frozen_stack(depth=3, d=512):
    torch.manual_seed(0)
    model = torch.nn.Sequential(*[torch.nn.Linear(d, d) for _ in range(depth)]).to(DEV, BF16)
    q.quantize(model, weights=q.qint8, activations=q.qint8)
    q.freeze(model)
    return model


@pytest.mark.parametrize("streamline", [True, False])
def test_calibration_forward_does_not_synchronise(streamline):
    model = frozen_stack()
    xs = batches((8, 512), k=3)
    with torch.no_grad():
        with q.Calibration(streamline=streamline):
            frozen_stack()(xs[0])  # first use of each kernel and buffer outside the checked region
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for x in xs:
                with q.Calibration(streamline=streamline):
                    model(x)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    assert all(not torch.all(m.output_scale == 1) for m in model if isinstance(m, q.QModuleMixin))


def test_calibration_step_replays_in_a_cuda_graph():
    eager, graphed = frozen_stack(), frozen_stack()
    xs = batches((16, 512), k=6, seed=3)
    cal = q.Calibration()
    with torch.no_grad():
        for model in (eager, graphed):
            with q.Calibration():
                model(xs[0])
        static = xs[0].clone()
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph), cal:
            graphed(static)
        for x in xs[1:]:
            with q.Calibration():
                eager(x)
            static.copy_(x)
            graph.replay()
    torch.cuda.synchronize()
    assert_same_scales(eager, graphed)


# the softmax takes the float output of the first bmm, so quanto::qbytes_softmax does not run in this block
ONE_LAUNCH_OPS = ("qbytes_linear_quantized", "qbytes_layer_norm", "qbytes_bmm")


def count_calls(monkeypatch):
    calls = dict.fromkeys(ONE_LAUNCH_OPS, 0)
    for name in ONE_LAUNCH_OPS:
        def counted(*args, _op=getattr(torch.ops.quanto, name), _name=name, **kwargs):
            calls[_name] += 1
            return _op(*args, **kwargs)
        monkeypatch.setattr(torch.ops.quanto, name, counted)
    return calls


def test_fused_paths_stand_aside_while_calibrating(monkeypatch):
    model = frozen_encoder()
    x = batches((2, 16, 64), k=1)[0]
    calls = count_calls(monkeypatch)
    with torch.no_grad(), q.Calibration(streamline=False):
        model(x)
    assert calls["qbytes_linear_quantized"] == 0 and calls["qbytes_layer_norm"] == 0, calls
    with torch.no_grad():
        model(x)
    assert calls["qbytes_linear_quantized"] > 0 and calls["qbytes_layer_norm"] == 2, calls


def test_quantize_calibrate_freeze_requantize_round_trip(monkeypatch):
    torch.manual_seed(0)
    model = Encoder().to(DEV, BF16)
    q.quantize(model, weights=q.qint8, activations=q.qint8)
    with torch.no_grad():
        for x in batches((2, 16, 64), k=3, seed=7):
            with q.Calibration(streamline=False):
                model(x)
    q.freeze(model)
    state = model.state_dict()
    qmap = q.quantization_map(model)
    with torch.device("meta"):
        fresh = Encoder().to(BF16)
    q.requantize(fresh, state, qmap, device=DEV)
    assert q.quantization_map(fresh) == qmap
    for name, m in fresh.named_modules():
        if isinstance(m, q.QModuleMixin):
            ref = model.get_submodule(name)
            assert torch.equal(m.input_scale, ref.input_scale) and torch.equal(m.output_scale, ref.output_scale)
            assert m.frozen == ref.frozen
    x = batches((2, 16, 64), k=1, seed=11)[0]
    calls = count_calls(monkeypatch)
    with torch.no_grad():
        y0 = model(x)
        y1 = fresh(x)
    assert torch.equal(y0, y1)
    # after calibration the one-launch paths run again, in both models
    assert all(calls[name] > 0 and calls[name] % 2 == 0 for name in ONE_LAUNCH_OPS), calls
