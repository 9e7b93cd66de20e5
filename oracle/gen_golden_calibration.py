"""Write tests/golden/calibration.npz from the REAL reference on CPU (needs the reference installed in oracle/_ref by
oracle/build_ref.py): its Calibration scale update (optimum/quanto/calibrate.py:31-34 `_updated_scale` of 37-61
`absmax_scale`), and the streamline decisions and quantization_map of two small models.

    python oracle/gen_golden_calibration.py

Op sequences: case `c` stores c_meta = [T code (0 f32, 1 f16, 2 bf16), qmax, momentum, steps], c_s = the scale bits
before the first step and after every step (uint32 for f32, uint16 for f16 / bf16), and c_x<j> = the bits of the
tensor of step j.  The scale starts at 1 (a fresh module's buffer).

Models: `<model>_<streamline>_live` lists, in `<model>_names` order, whether each quantized module's output hook is
still registered after one calibrated forward; `<model>_map` is the JSON of quantization_map(model).
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

from optimum.quanto import Calibration, qfloat8_e4m3fn, qfloat8_e4m3fnuz, qfloat8_e5m2, qint8, quantization_map, quantize  # noqa: E402,E501
from optimum.quanto.calibrate import _updated_scale, absmax_scale  # noqa: E402

DT = [torch.float32, torch.float16, torch.bfloat16]
QT = {"int8": qint8, "e4m3fn": qfloat8_e4m3fn, "e5m2": qfloat8_e5m2, "e4m3fnuz": qfloat8_e4m3fnuz}
MOMENTA = (0.9, 0.5, 0.99)
SIZES = (1, 7, 33, 130, 515)
MAGNITUDES = (1.0, 0.1, 3.0, 10.0, 0.01, 250.0)


def bits(t):
    t = t.detach().contiguous()
    if t.dtype == torch.float32:
        return t.view(torch.int32).numpy().view(np.uint32)
    return t.view(torch.int16).numpy().view(np.uint16)


def sequences(gen, dt, qt):
    """The step tensors of each sequence kind: ordinary batches, a first batch whose scale comes out exactly 1 (so the
    next batch replaces it again), and batches holding a NaN and an inf."""
    qmax = torch.finfo(qt.dtype).max if qt.dtype.is_floating_point else torch.iinfo(qt.dtype).max

    def batch(j):
        n = SIZES[j % len(SIZES)]
        return (torch.randn(n, generator=gen) * MAGNITUDES[j % len(MAGNITUDES)]).to(dt)

    plain = [batch(j) for j in range(6)]
    first = batch(1)
    first[first.numel() // 2] = -qmax  # max |x| == qmax: the first scale is exactly 1
    reset = [first] + [batch(j) for j in range(2, 5)]
    nan = [batch(0), batch(2)]
    nan[1][3 % nan[1].numel()] = float("nan")
    nan.append(batch(3))
    inf = [batch(0), batch(3)]
    inf[1][5 % inf[1].numel()] = float("-inf")
    inf.append(batch(4))
    first_inf = [batch(2)]
    first_inf[0][0] = float("inf")
    first_inf.append(batch(1))
    return [plain, reset, nan, inf, first_inf]


def op_cases(out):
    gen = torch.Generator().manual_seed(0)
    c = 0
    for code, dt in enumerate(DT):
        for qt in QT.values():
            for momentum in MOMENTA:
                for seq in sequences(gen, dt, qt):
                    scale = torch.ones((), dtype=dt)
                    scales = [bits(scale)]
                    for j, x in enumerate(seq):
                        scale = _updated_scale(scale, absmax_scale(x, qt), momentum)
                        assert scale.dtype == dt
                        scales.append(bits(scale))
                        out[f"{c}_x{j}"] = bits(x)
                    qmax = float(torch.finfo(qt.dtype).max if qt.dtype.is_floating_point else 127)
                    out[f"{c}_meta"] = np.array([code, qmax, momentum, len(seq)], dtype=np.float64)
                    out[f"{c}_s"] = np.stack(scales)
                    c += 1
    return c


class MLP3(torch.nn.Module):
    """l3(silu(l2(l1(x))))"""

    def __init__(self, d=32):
        super().__init__()
        self.l1 = torch.nn.Linear(d, 64)
        self.l2 = torch.nn.Linear(64, 64)
        self.l3 = torch.nn.Linear(64, d)

    def forward(self, x):
        return self.l3(torch.nn.functional.silu(self.l2(self.l1(x))))


class Encoder(torch.nn.Module):
    """A single-head pre-LN encoder block: Linear, LayerNorm, bmm and softmax."""

    def __init__(self, d=32):
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


def live(m):
    handle = m._quantize_hooks.get("output")
    return handle is not None and handle.id in m._forward_hooks


def model_cases(out):
    for tag, cls, shape in (("mlp3", MLP3, (4, 32)), ("encoder", Encoder, (2, 8, 32))):
        names = None
        for streamline in (True, False):
            torch.manual_seed(1)
            model = cls()
            quantize(model, weights=qint8, activations=qint8)
            x = torch.randn(shape)
            with torch.no_grad(), Calibration(streamline=streamline):
                model(x)
            qmods = [(n, m) for n, m in model.named_modules() if hasattr(m, "_quantize_hooks")]
            names = [n for n, _ in qmods]
            out[f"{tag}_{int(streamline)}_live"] = np.array([live(m) for _, m in qmods])
            out[f"{tag}_map"] = np.array(json.dumps(quantization_map(model), sort_keys=True))
        out[f"{tag}_names"] = np.array(names)


def main():
    out = {}
    n = op_cases(out)
    model_cases(out)
    path = os.path.join(ROOT, "tests", "golden", "calibration.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {n} op sequences", {k: out[k] for k in out if k.endswith("_live")})


if __name__ == "__main__":
    main()
