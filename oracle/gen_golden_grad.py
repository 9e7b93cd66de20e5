"""Generate tests/golden/grad.npz from the REAL reference's autograd (huggingface/optimum-quanto, CPU path).

Run in the authoring container only (the reference cannot travel to the GPU box):

    PYTHONPATH=/root/reference python oracle/gen_golden_grad.py

A separate script and seed next to oracle/gen_golden.py (whose fixtures it leaves untouched); it reuses that script's
bit-pattern conventions.  The fixture pins oracle/grad_oracle.py (tests/test_grad_oracle.py) and is replayed against the
CUDA backward (tests/test_gpu_grad.py::test_fixture_replay).
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gen_golden import OUT, TAG, bits  # noqa: E402  (imports optimum.quanto, registers torch.ops.quanto.*)
from optimum.quanto import qfloat8_e4m3fn, qint4, qint8  # noqa: E402


def gen_grad(g):
    """Backward of QLinear through the reference's own autograd (tests/nn/test_qlinear.py::test_qlinear_gradient):
    qint4 (group 128, bf16 and fp16), qint8 and qfloat8_e4m3fn weights, frozen (weight.requires_grad False, the adapter
    fine-tuning case) and unfrozen (quantization-aware training).  Stores the seeded gO, the reference's input.grad,
    bias.grad and (unfrozen) weight.grad, and the quantized weight the frozen layer used.  Its own file and seed: the
    fixtures committed earlier stay byte-identical."""
    from optimum.quanto.nn import QLinear

    cases = {}
    idx = 0
    for dtype, wq, K, N, M in [
        (torch.bfloat16, qint4, 256, 128, 12),
        (torch.float16, qint4, 256, 128, 12),
        (torch.bfloat16, qint8, 128, 64, 8),
        (torch.float16, qfloat8_e4m3fn, 128, 64, 8),
    ]:
        for frozen in (True, False):
            lin = torch.nn.Linear(K, N, bias=True).to(dtype)
            with torch.no_grad():
                lin.weight.copy_((torch.randn(N, K, generator=g) * 0.05).to(dtype))
                lin.bias.copy_((torch.randn(N, generator=g) * 0.1).to(dtype))
            q = QLinear.from_module(lin, weights=wq)
            if frozen:
                qw = q.qweight  # canonical tensors, as in gen_qlinear
                if type(qw).__name__ not in ("WeightQBytesTensor", "WeightQBitsTensor"):
                    qw = qw.weight_qbits_tensor() if hasattr(qw, "weight_qbits_tensor") else qw.weight_qbytes_tensor()
                q.weight = torch.nn.Parameter(qw, requires_grad=False)
            x = torch.randn(M, K, generator=g).to(dtype).requires_grad_(True)
            y = q(x)
            gO = torch.randn(M, N, generator=g).to(dtype)
            y.backward(gO)
            p = f"g{idx}_"
            cases[p + "tag"] = np.array(TAG[dtype])
            cases[p + "wq"] = np.array(wq.name)
            cases[p + "frozen"] = np.int64(frozen)
            cases[p + "shape"] = np.array([N, K, M, q.weight_group_size or 0], dtype=np.int64)
            cases[p + "bias"] = bits(lin.bias)
            cases[p + "x"] = bits(x)
            cases[p + "gO"] = bits(gO)
            cases[p + "x_grad"] = bits(x.grad)
            cases[p + "bias_grad"] = bits(q.bias.grad)
            if frozen:
                for k, v in q.state_dict().items():
                    if k.startswith("weight"):
                        cases[p + "sd_" + k] = bits(v)
            else:
                cases[p + "weight"] = bits(lin.weight)
                cases[p + "weight_grad"] = bits(q.weight.grad)
            idx += 1
    cases["n"] = np.int64(idx)
    np.savez_compressed(os.path.join(OUT, "grad.npz"), **cases)



def main():
    torch.set_num_threads(1)  # deterministic accumulation order for the stored float results
    gen_grad(torch.Generator().manual_seed(20261018))
    print("wrote", os.path.normpath(os.path.join(OUT, "grad.npz")))
    return 0


if __name__ == "__main__":
    sys.exit(main())
