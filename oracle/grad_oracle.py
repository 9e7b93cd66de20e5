"""Input gradient of the quantized linear, restated on the numpy oracle (oracle/quanto_oracle.py).

TEST INFRASTRUCTURE ONLY, like quanto_oracle.py.  Pinned by tests/test_grad_oracle.py against tests/golden/grad.npz,
which oracle/gen_golden_grad.py produces from the real reference's autograd.
"""
import numpy as np

from . import quanto_oracle as O


def grad_input_from_dequantized(g_f32: np.ndarray, w_f32: np.ndarray, tag: str = "bf16"):
    """Input gradient of the quantized linear -- QuantizedLinearFunction.backward, optimum/quanto/tensor/function.py:49-63:
    g_in = torch.matmul(gO, other) with `other` dequantised by qfallback (O.dequantize_qbits for int4; rnd(scale * W)
    for 8-bit weights, tensor/qbytes.py:23-31).  gO [M, N], w [N, K] (the dequantised weight).

    Returns (dx_exact_f64, dx_rounded_storage, tol) as O.linear_from_dequantized does (no bias)."""
    return O.linear_from_dequantized(g_f32, np.asarray(w_f32).T, None, tag)
