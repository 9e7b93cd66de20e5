"""CPU checks of calibration and the model API: the numpy oracle of the scale update against the reference's own op
sequences (tests/golden/calibration.npz), the fake of quanto::absmax_update_ and its argument checks, and quantize /
quantization_map / requantize on CPU modules (the cases of the reference's tests/quantize/test_quantize_patterns.py)."""
import json
import os

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

import quanto_b200 as q
from oracle import calibration_oracle as CO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "calibration.npz")


def same_bits(got, want, tag):
    """Equal bit patterns, or both NaN (the NaN payload is not part of the contract)."""
    return got == want or (np.isnan(CO.values(np.array([got]), tag)[0]) and np.isnan(CO.values(np.array([want]), tag)[0]))


def test_oracle_reproduces_every_golden_scale():
    g = np.load(GOLDEN)
    n = sum(1 for k in g.files if k.endswith("_meta"))
    assert n == 3 * 4 * 3 * 5
    steps = 0
    for c in range(n):
        code, qmax, momentum, count = g[f"{c}_meta"]
        tag = CO.TAGS[int(code)]
        s = g[f"{c}_s"]
        assert CO.values(s[:1], tag)[0] == 1
        scale = CO.values(s[:1], tag)[0]
        for j in range(int(count)):
            scale = CO.absmax_update(scale, CO.values(g[f"{c}_x{j}"], tag), qmax, momentum, tag)
            got = CO.bits_of(np.array([scale], np.float32), tag)[0]
            assert same_bits(got, s[j + 1], tag), (c, j, tag, qmax, momentum, hex(got), hex(s[j + 1]))
            steps += 1
    assert steps == 648


def test_golden_covers_the_update_rules():
    """The fixture holds first batches, a later scale of exactly 1 (replaced again), NaN and inf scales."""
    g = np.load(GOLDEN)
    n = sum(1 for k in g.files if k.endswith("_meta"))
    ones_after_first = nans = infs = 0
    for c in range(n):
        tag = CO.TAGS[int(g[f"{c}_meta"][0])]
        v = CO.values(g[f"{c}_s"], tag)
        ones_after_first += int(v[1] == 1 and v[2] != 1)
        nans += int(np.isnan(v).any())
        infs += int(np.isinf(v).any())
    assert ones_after_first == 36 and nans >= 36 and infs >= 36


# ------------------------------------------------------------------------------------- quanto::absmax_update_ fake
def test_fake_runs_under_fake_tensor_mode():
    with FakeTensorMode():
        for dt in (torch.float32, torch.float16, torch.bfloat16):
            scale = torch.ones((), dtype=dt, device="cuda")
            x = torch.empty(3, 5, dtype=dt, device="cuda")
            assert torch.ops.quanto.absmax_update_(scale, x, 127.0, 0.9) is None


@pytest.mark.parametrize("case", ["empty", "mismatch", "int", "shape", "qmax", "device"])
def test_fake_rejects_what_the_op_rejects(case):
    scale_shape, scale_dtype, n, dtype, qmax = (), torch.bfloat16, 4, torch.bfloat16, 127.0
    if case == "empty":
        n = 0
    elif case == "mismatch":
        scale_dtype = torch.float32
    elif case == "int":
        scale_dtype = dtype = torch.int8
    elif case == "shape":
        scale_shape = (2,)
    elif case == "qmax":
        qmax = 0.0
    with FakeTensorMode():
        scale = torch.empty(scale_shape, dtype=scale_dtype, device="cuda")
        x = torch.empty(n, dtype=dtype, device="cpu" if case == "device" else "cuda")
        with pytest.raises(ValueError):
            torch.ops.quanto.absmax_update_(scale, x, qmax, 0.9)


def test_calibrating_follows_the_mode():
    from quanto_b200.calibrate import calibrating

    assert not calibrating()
    with q.Calibration():
        assert calibrating()
        with q.Calibration(streamline=False):
            assert calibrating()
        assert calibrating()
    assert not calibrating()


def test_calibration_constructor_and_enter():
    cal = q.Calibration()
    assert (cal.momentum, cal.streamline, cal.debug) == (0.9, True, False)
    cal = q.Calibration(momentum=0.5, streamline=False, debug=True)
    assert (cal.momentum, cal.streamline, cal.debug) == (0.5, False, True)
    with cal as entered:
        assert entered is None


# ------------------------------------------------------------------------ quantize: include / exclude patterns
# The cases of the reference's test_quantize_patterns.py on a model of the same shape: a child module holding three
# leaves, and a head beside it.
class Trunk(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.embed = torch.nn.Linear(24, 40)
        self.hidden = torch.nn.Linear(40, 40)
        self.proj = torch.nn.Linear(40, 12)


class Net(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.trunk = Trunk()
        self.head = torch.nn.Linear(12, 3)


LEAVES = ("trunk.embed", "trunk.hidden", "trunk.proj", "head")


def quantized_names(model):
    return {name for name, m in model.named_modules() if isinstance(m, q.QModuleMixin)}


@pytest.mark.parametrize("leaf", LEAVES)
def test_quantize_includes_one_leaf(leaf):
    model = Net()
    q.quantize(model, weights=q.qint8, include=leaf)
    assert quantized_names(model) == {leaf}


@pytest.mark.parametrize("leaf", LEAVES)
def test_quantize_excludes_one_leaf(leaf):
    model = Net()
    q.quantize(model, weights=q.qint8, exclude=leaf)
    assert quantized_names(model) == set(LEAVES) - {leaf}


def test_quantize_include_and_exclude_by_prefix():
    model = Net()
    q.quantize(model, weights=q.qint8, include="trunk*")
    assert quantized_names(model) == {"trunk.embed", "trunk.hidden", "trunk.proj"}
    model = Net()
    q.quantize(model, weights=q.qint8, exclude=["trunk*"])
    assert quantized_names(model) == {"head"}
    model = Net()
    q.quantize(model, weights=q.qint8, include=["trunk.*", "head"], exclude="*.hidden")
    assert quantized_names(model) == {"trunk.embed", "trunk.proj", "head"}


class Mixed(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(3, 8, 3)
        self.norm = torch.nn.LayerNorm(8)
        self.block = torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.GELU(), torch.nn.Linear(16, 4, bias=False))


def test_quantize_swaps_modules_and_drops_parameters():
    model = Mixed()
    originals = dict(model.named_modules())
    weights = {n: m.weight for n, m in originals.items() if getattr(m, "weight", None) is not None}
    q.quantize(model, weights=q.qint4)
    assert isinstance(model.conv, q.QConv2d) and isinstance(model.block[0], q.QLinear)
    assert isinstance(model.block[2], q.QLinear) and model.block[2].bias is None
    assert type(model.norm) is torch.nn.LayerNorm  # a LayerNorm is quantized only with activations
    assert isinstance(model.block[1], torch.nn.GELU)
    for name in ("conv", "block.0", "block.2"):
        qm = model.get_submodule(name)
        assert qm.name == name and qm.weight_qtype is q.qint4 and qm.activation_qtype is None
        assert qm.weight is weights[name]  # the quantized module took the tensor over
        assert originals[name].weight is None
    assert originals["norm"].weight is not None
    assert q.quantization_map(model) == {n: {"weights": "qint4", "activations": "none"}
                                         for n in ("conv", "block.0", "block.2")}


def test_quantize_with_activations_and_string_qtypes():
    model = Mixed()
    q.quantize(model, weights="qint8", activations="qfloat8_e4m3fn", exclude="conv")
    assert isinstance(model.norm, q.QLayerNorm) and type(model.conv) is torch.nn.Conv2d
    assert model.norm.weight_qtype is None and model.norm.activation_qtype is q.qfloat8_e4m3fn
    assert q.quantization_map(model) == {
        "norm": {"weights": "none", "activations": "qfloat8_e4m3fn"},
        "block.0": {"weights": "qint8", "activations": "qfloat8_e4m3fn"},
        "block.2": {"weights": "qint8", "activations": "qfloat8_e4m3fn"},
    }
    assert q.quantize_module(torch.nn.ReLU(), weights=q.qint8) is None
    assert q.quantize_module(torch.nn.LayerNorm(4), weights=q.qint8) is None


def test_quantization_map_matches_the_reference():
    """The fixture's quantization maps, from the reference's quantize() of the same two models."""
    g = np.load(GOLDEN)
    assert json.loads(str(g["mlp3_map"])) == {n: {"weights": "qint8", "activations": "qint8"} for n in ("l1", "l2", "l3")}
    enc = json.loads(str(g["encoder_map"]))
    assert sorted(enc) == sorted(str(n) for n in g["encoder_names"])
    for name, v in enc.items():  # a QLayerNorm never quantizes its weight
        assert v == {"weights": "none" if name.startswith("ln") else "qint8", "activations": "qint8"}, name


def test_requantize_unfrozen_state_dict_into_a_meta_model():
    torch.manual_seed(0)
    model = Mixed()
    q.quantize(model, weights=q.qint8, activations=q.qint8)
    model.norm.output_scale.fill_(0.25)
    model.block[0].input_scale.fill_(0.5)
    sd = model.state_dict()
    with torch.device("meta"):
        fresh = Mixed()
    q.requantize(fresh, sd, q.quantization_map(model))
    assert q.quantization_map(fresh) == q.quantization_map(model)
    for (n, a), (_, b) in zip(model.state_dict().items(), fresh.state_dict().items()):
        assert b.device.type == "cpu" and torch.equal(a, b), n
    assert fresh.norm.output_scale.item() == 0.25 and fresh.block[0].input_scale.item() == 0.5
