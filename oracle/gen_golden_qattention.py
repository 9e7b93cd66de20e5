"""Write tests/golden/qattention.npz from the REAL reference on CPU (needs the reference installed in oracle/_ref
by oracle/build_ref.py): the reference's ActivationQBytesTensor bmm (qbytes_ops.py:175-186) and _softmax (:208-215).

    python oracle/gen_golden_qattention.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref"))

from optimum.quanto import qfloat8_e4m3fn, qfloat8_e4m3fnuz, qfloat8_e5m2, qint8  # noqa: E402
from optimum.quanto.tensor.activations.qbytes import ActivationQBytesTensor  # noqa: E402

DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}
QT = {"int8": qint8, "e4m3fn": qfloat8_e4m3fn, "e5m2": qfloat8_e5m2, "e4m3fnuz": qfloat8_e4m3fnuz}


def bits(t):
    t = t.contiguous()
    if t.dtype == torch.float32:
        return t.numpy()
    if t.dtype in (torch.float16, torch.bfloat16):
        return t.view(torch.int16).numpy().view(np.uint16)
    if t.dtype == torch.int8:
        return t.numpy()
    return t.view(torch.uint8).numpy()


def act(qtype, data, scale):
    return ActivationQBytesTensor(qtype, data.size(), data.stride(), data, scale)


def main():
    gen = torch.Generator().manual_seed(0)
    out = {}
    # bmm: the reference's own test shape (K = 10, N = 6) and a tensor-core one
    a = torch.randint(-128, 128, (3, 5, 10), dtype=torch.int8, generator=gen)
    b = torch.randint(-128, 128, (3, 10, 6), dtype=torch.int8, generator=gen)
    out["bmm_a"], out["bmm_b"] = a.numpy(), b.numpy()
    out["bmm_sa"], out["bmm_sb"] = np.float32(0.0123), np.float32(0.0456)
    for tag, dt in DT.items():
        y = torch.bmm(act(qint8, a, torch.tensor(0.0123, dtype=dt)), act(qint8, b, torch.tensor(0.0456, dtype=dt)))
        out[f"bmm_out_{tag}"] = bits(y)
    # softmax: 4 rows of 37 codes of every 8-bit qtype
    out["sm_scale"] = np.float32(0.0625)
    for q_tag, qt in QT.items():
        if q_tag == "int8":
            codes = torch.randint(-127, 128, (4, 37), dtype=torch.int8, generator=gen)
        else:
            codes = (torch.randn(4, 37, generator=gen) * 3).to(qt.dtype)
        out[f"sm_in_{q_tag}"] = bits(codes)
        for tag in ("f32", "bf16"):
            y = torch.softmax(act(qt, codes, torch.tensor(0.0625, dtype=DT[tag])), dim=-1)
            assert isinstance(y, ActivationQBytesTensor)
            out[f"sm_out_{q_tag}_{tag}"] = bits(y._data)
            out[f"sm_scale_out_{q_tag}_{tag}"] = bits(y._scale.reshape(()))
    path = os.path.join(ROOT, "tests", "golden", "qattention.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, sorted(out))


if __name__ == "__main__":
    main()
