"""Write tests/golden/qlayernorm.npz from the REAL reference on CPU (needs the reference installed in oracle/_ref by
oracle/build_ref.py): its QLayerNorm (optimum/quanto/nn/qlayernorm.py) with the quantize_output hook
(nn/qmodule.py:296-302), from float inputs and from ActivationQBytesTensor inputs (dequantized by qfallback).

    python oracle/gen_golden_qlayernorm.py

Case `c` stores c_x (input: float bits, or codes with c_sin the input scale), c_w / c_b (absent when the module has
none), c_s (output scale bits; float32 for the non-affine module, whose scale dtype is float32), c_out (the codes) and
c_meta = [T, qtype, affine, input kind, H, eps].
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

from optimum.quanto import qfloat8_e4m3fn, qfloat8_e4m3fnuz, qfloat8_e5m2, qint8  # noqa: E402
from optimum.quanto.nn import QLayerNorm  # noqa: E402
from optimum.quanto.tensor.activations.qbytes import ActivationQBytesTensor  # noqa: E402

DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
QT = {"int8": qint8, "e4m3fn": qfloat8_e4m3fn, "e5m2": qfloat8_e5m2, "e4m3fnuz": qfloat8_e4m3fnuz}
AFFINE = {"affine": (True, True), "weight": (True, False), "none": (False, False)}


def bits(t):
    t = t.detach().contiguous()
    if t.dtype == torch.float32:
        return t.numpy()
    if t.dtype in (torch.float16, torch.bfloat16):
        return t.view(torch.int16).numpy().view(np.uint16)
    if t.dtype == torch.int8:
        return t.numpy()
    return t.view(torch.uint8).numpy()


def main():
    gen = torch.Generator().manual_seed(0)
    out = {}
    i = 0
    for tag, dt in DT.items():
        for q_tag, qt in QT.items():
            for kind, (affine, has_bias) in AFFINE.items():
                for src in ("float", "codes"):
                    for h in (1, 32, 50, 768):
                        if h == 768 and (kind != "affine" or (src == "codes") != (q_tag in ("e4m3fn", "e4m3fnuz"))):
                            continue  # one wide row per (T, qtype), both input forms among them: a small fixture
                        rows = 1 if h == 768 else 3
                        norm = torch.nn.LayerNorm(h, elementwise_affine=affine, bias=has_bias).to(dt)
                        with torch.no_grad():
                            if norm.weight is not None:
                                norm.weight.copy_(1 + 0.5 * torch.randn(h, generator=gen))
                            if norm.bias is not None:
                                norm.bias.copy_(0.5 * torch.randn(h, generator=gen))
                        qnorm = QLayerNorm.from_module(norm, activations=qt)
                        x = (torch.randn(rows, h, generator=gen) * 2 + 0.5).to(dt)
                        if src == "codes":
                            s_in = torch.tensor(0.05, dtype=dt)
                            data = torch.ops.quanto.quantize_symmetric(x, qt.dtype, None, s_in)
                            inp = ActivationQBytesTensor(qt, data.size(), data.stride(), data, s_in)
                            out[f"{i}_x"], out[f"{i}_sin"] = bits(data), bits(s_in)
                        else:
                            inp = x
                            out[f"{i}_x"] = bits(x)
                        # an output scale that saturates the largest outputs of the row
                        qmax = float(torch.finfo(qt.dtype).max if qt.dtype.is_floating_point else 127)
                        s_out = torch.tensor(3.0 / qmax, dtype=qnorm.output_scale.dtype)
                        qnorm.output_scale = s_out
                        with torch.no_grad():
                            y = qnorm(inp)
                        assert isinstance(y, ActivationQBytesTensor) and y.qtype is qt
                        if norm.weight is not None:
                            out[f"{i}_w"] = bits(norm.weight)
                        if norm.bias is not None:
                            out[f"{i}_b"] = bits(norm.bias)
                        out[f"{i}_s"] = bits(s_out)
                        out[f"{i}_out"] = bits(y._data)
                        out[f"{i}_meta"] = np.array([tag, q_tag, kind, src, str(h), repr(norm.eps)])
                        i += 1
    for kind, (affine, has_bias) in AFFINE.items():
        qnorm = QLayerNorm.from_module(torch.nn.LayerNorm(32, elementwise_affine=affine, bias=has_bias), activations=qint8)
        sd = qnorm.state_dict()
        out[f"sd_keys_{kind}"] = np.array(list(sd.keys()))
        out[f"sd_none_{kind}"] = np.array([k for k, v in sd.items() if v is None] or [""])
        out[f"sd_dtypes_{kind}"] = np.array([str(v.dtype) for v in sd.values() if v is not None])
    out["cases"] = np.int64(i)
    path = os.path.join(ROOT, "tests", "golden", "qlayernorm.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, i, "cases")


if __name__ == "__main__":
    main()
