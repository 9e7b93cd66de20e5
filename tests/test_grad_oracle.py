"""CPU: the input-gradient restatement of the oracle (oracle/grad_oracle.py) against the reference's own autograd
(tests/golden/grad.npz, written by oracle/gen_golden_grad.py), and the schemas of the input-gradient ops."""
import os

import numpy as np
import torch

import quanto_b200  # noqa: F401  (registers torch.ops.quanto.*)
from oracle import grad_oracle as GO
from oracle import quanto_oracle as O


def _dequantized_weight(z, p, tag):
    """The dequantised weight the frozen reference layer multiplied with (qfallback -> dequantize())."""
    N, K, _, G = (int(v) for v in z[p + "shape"])
    wq = str(z[p + "wq"])
    if wq == "qint4":
        deq = O.dequantize_qbits(z[p + "sd_weight._data._data"], 4, z[p + "sd_weight._scale"],
                                 z[p + "sd_weight._shift"], tag, N, K, G)
        return O.to_f32(deq, tag)
    data = z[p + "sd_weight._data"]
    w = data.astype(np.float32) if wq == "qint8" else O.fp8_bits_to_f32(data, "e4m3fn")
    s = O.to_f32(z[p + "sd_weight._scale"], tag).reshape(-1, 1)
    return O.round_to(s * w, tag)


def test_grad_input_oracle_matches_reference_autograd(golden_dir):
    z = np.load(os.path.join(golden_dir, "grad.npz"))
    checked = 0
    for i in range(int(z["n"])):
        p = f"g{i}_"
        tag = str(z[p + "tag"])
        gO = O.to_f32(z[p + "gO"], tag)
        # bias.grad = gO summed over the rows, rounded once (both layers)
        b64 = gO.astype(np.float64).sum(axis=0)
        bref = O.to_f32(z[p + "bias_grad"], tag).astype(np.float64)
        assert np.all(np.abs(bref - b64) <= 0.5 * O.ulp(b64, tag) + 2.0 ** -20 * np.abs(gO).sum(axis=0)), i
        if not int(z[p + "frozen"]):
            continue
        wd = _dequantized_weight(z, p, tag)
        dx64, dx_round, tol = GO.grad_input_from_dequantized(gO, wd, tag)
        ref = O.to_f32(z[p + "x_grad"], tag).astype(np.float64)
        bound = 1.02 * tol + O.accumulate_allowance(gO, wd.T)
        assert np.all(np.abs(ref - dx64) <= bound), (i, float(np.max(np.abs(ref - dx64) / bound)))
        rel = np.linalg.norm(O.to_f32(dx_round, tag) - ref) / np.linalg.norm(ref)
        assert rel < 1e-3, (i, rel)
        checked += 1
    assert checked == 4


def test_grad_input_oracle_is_the_transposed_linear():
    rng = np.random.default_rng(3)
    g = O.round_to(rng.standard_normal((5, 48)).astype(np.float32), "bf16")
    w = O.round_to(rng.standard_normal((48, 32)).astype(np.float32), "bf16")
    dx64, _, _ = GO.grad_input_from_dequantized(g, w, "bf16")
    assert np.allclose(dx64, g.astype(np.float64) @ w.astype(np.float64), rtol=0, atol=0)


def test_grad_input_ops_registered():
    s = str(torch.ops.quanto.qbits_grad_input.default._schema)
    assert ("Tensor grad_output, Tensor packed, Tensor scale, Tensor shift, int out_features, int group_size, int bits"
            in s), s
    s = str(torch.ops.quanto.qbytes_grad_input.default._schema)
    assert "Tensor grad_output, Tensor B, Tensor scales" in s, s
