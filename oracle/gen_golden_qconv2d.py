"""Write tests/golden/qconv2d.npz from the REAL reference on CPU (needs the reference installed in oracle/_ref by
oracle/build_ref.py): its QConv2d (optimum/quanto/nn/qconv2d.py) quantized to qint4 (groups 96 and 128), qint8 and
qfloat8, frozen on the canonical classes (not TinyGemm: SURVEY 8c), and its outputs.

    python oracle/gen_golden_qconv2d.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

from optimum.quanto import qfloat8_e4m3fn, qint4, qint8  # noqa: E402
from optimum.quanto.nn import QConv2d  # noqa: E402

# (weights, Cin, Cout, kernel, stride, padding, dilation, input [B, H, W]); group = the reference's pick for Cin*kh*kw
CASES = [
    (qint4, 32, 16, 3, 1, 1, 1, (2, 6, 6)),      # K = 288 -> group 96
    (qint4, 128, 16, 3, 2, 1, 1, (1, 7, 5)),     # K = 1152 -> group 128
    (qint8, 16, 32, 3, 1, 1, 2, (2, 7, 6)),
    (qfloat8_e4m3fn, 16, 32, 1, 1, 0, 1, (2, 5, 5)),
]


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
    g = torch.Generator().manual_seed(0)
    out = {}
    dtype = torch.bfloat16
    for i, (wq, cin, cout, k, s, p, d, (b, h, w)) in enumerate(CASES):
        conv = torch.nn.Conv2d(cin, cout, k, stride=s, padding=p, dilation=d, bias=True)
        with torch.no_grad():
            conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) * 0.05)
            conv.bias.copy_(torch.randn(cout, generator=g) * 0.1)
        conv = conv.to(dtype)
        qc = QConv2d.from_module(conv, weights=wq)
        qw = qc.qweight
        if type(qw).__name__ not in ("WeightQBytesTensor", "WeightQBitsTensor"):
            qw = qw.weight_qbits_tensor() if hasattr(qw, "weight_qbits_tensor") else qw.weight_qbytes_tensor()
        qc.weight = torch.nn.Parameter(qw, requires_grad=False)
        x = torch.randn(b, cin, h, w, generator=g).to(dtype)
        with torch.no_grad():
            y = qc(x)
        pre = f"c{i}_"
        out[pre + "wq"] = np.array(wq.name)
        out[pre + "geom"] = np.array([cin, cout, k, s, p, d, qc.weight_group_size or 0], dtype=np.int64)
        out[pre + "w"] = bits(conv.weight)
        out[pre + "bias"] = bits(conv.bias)
        out[pre + "x"] = bits(x)
        for key, v in qc.state_dict().items():
            if key.startswith("weight"):
                out[pre + "sd_" + key] = bits(v)
        out[pre + "y"] = bits(y)
    out["n"] = np.int64(len(CASES))
    path = os.path.join(ROOT, "tests", "golden", "qconv2d.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, sorted(out))


if __name__ == "__main__":
    main()
