"""CPU checks of the quantized conv2d: the im2col oracle (oracle/conv_oracle.py) pinned to the reference's QConv2d
fixture (tests/golden/qconv2d.npz, oracle/gen_golden_qconv2d.py), and the fakes of the two conv ops."""
import os

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from helpers import ROOT
from oracle import conv_oracle as CO
from oracle import quanto_oracle as O

import quanto_b200  # noqa: F401  (registers torch.ops.quanto.*)

GOLDEN = os.path.join(ROOT, "tests", "golden", "qconv2d.npz")


def test_im2col_matches_torch_unfold():
    x = np.random.default_rng(0).standard_normal((2, 3, 7, 6)).astype(np.float32)
    for kh, kw, s, p, d in ((3, 3, 1, 1, 1), (2, 3, 2, 0, 1), (3, 2, 1, 2, 2), (1, 1, 2, 0, 1)):
        cols, (b, ho, wo) = CO.im2col(x, kh, kw, (s, s), (p, p), (d, d))
        ref = torch.nn.functional.unfold(torch.from_numpy(x), (kh, kw), dilation=d, padding=p, stride=s)
        ref = ref.transpose(1, 2).reshape(-1, ref.shape[1]).numpy()  # unfold walks k as (c, r, s) too
        assert cols.shape == (b * ho * wo, 3 * kh * kw)
        assert np.array_equal(cols, ref)


def _dequantized(gold, pre, cout, k, group):
    wq = str(gold[pre + "wq"])
    scale = gold[pre + "sd_weight._scale"].reshape(-1)
    if wq == "qint4":
        shift = gold[pre + "sd_weight._shift"].reshape(-1)
        return O.to_f32(O.dequantize_qbits(gold[pre + "sd_weight._data._data"], 4, scale, shift, "bf16", cout, k, group),
                        "bf16").reshape(cout, k)
    data = gold[pre + "sd_weight._data"].reshape(cout, k)
    tag = "int8" if wq == "qint8" else "e4m3fn"
    w = data.astype(np.float32) if tag == "int8" else O.to_f32(data, tag)
    return O.to_f32(O.from_f32(w * O.to_f32(scale, "bf16").reshape(-1, 1), "bf16"), "bf16")


def test_conv_oracle_pins_reference_fixture():
    gold = np.load(GOLDEN)
    for i in range(int(gold["n"])):
        pre = f"c{i}_"
        cin, cout, k, s, p, d, group = (int(e) for e in gold[pre + "geom"])
        kk = cin * k * k
        w = _dequantized(gold, pre, cout, kk, group or kk).reshape(cout, cin, k, k)
        x = O.to_f32(gold[pre + "x"], "bf16")
        bias = O.to_f32(gold[pre + "bias"], "bf16")
        y64, y_ref, tol, cols = CO.conv_from_dequantized(x, w, bias, "bf16", (s, s), (p, p), (d, d))
        y = O.to_f32(gold[pre + "y"], "bf16").astype(np.float64)
        acc = CO.im2col(np.abs(x), k, k, (s, s), (p, p), (d, d))[0].astype(np.float64) @ np.abs(w).reshape(cout, -1).T
        acc = acc.reshape(y.shape[0], y.shape[2], y.shape[3], cout).transpose(0, 3, 1, 2)
        bound = 1.02 * tol + (2.0 ** -22) * np.sqrt(kk) * acc
        assert np.all(np.abs(y - y64) <= bound), (i, float(np.max(np.abs(y - y64) / bound)))
        # the reference's CPU convolution adds the bias to the fp32 sum and rounds once (what the sm_90a kernel does):
        # its output is the oracle's single rounding of the exact result, bit for bit
        assert np.array_equal(y, O.to_f32(y_ref, "bf16")), i


def test_conv_fakes():
    with FakeTensorMode():
        x = torch.empty(2, 32, 9, 7, dtype=torch.bfloat16, device="cuda")
        packed = torch.empty(64 * 3 // 2, 96, dtype=torch.uint8, device="cuda")
        coef = torch.empty(64 * 3, 1, dtype=torch.bfloat16, device="cuda")
        zp = torch.empty(64 * 3, 1, dtype=torch.uint8, device="cuda")
        bias = torch.empty(64, dtype=torch.bfloat16, device="cuda")
        y = torch.ops.quanto.qbits_conv2d(x, packed, coef, zp, bias, [64, 32, 3, 3], 96, 4, [2, 2], [1, 1], [1, 1])
        assert y.shape == (2, 64, 5, 4) and y.dtype == torch.bfloat16
        y = torch.ops.quanto.qbits_conv2d(x[0], packed, coef, coef, None, [64, 32, 3, 3], 96, 4, [1], [0], [2])
        assert y.shape == (64, 5, 3)
        w = torch.empty(64, 32, 3, 3, dtype=torch.float8_e4m3fn, device="cuda")
        s = torch.empty(64, 1, 1, 1, dtype=torch.bfloat16, device="cuda")
        y = torch.ops.quanto.qbytes_conv2d(x, w, s, bias, [1, 1], [1, 1], [1, 1])
        assert y.shape == (2, 64, 9, 7) and y.is_contiguous()
        with pytest.raises(ValueError):
            torch.ops.quanto.qbits_conv2d(x, packed, coef, coef, None, [64, 16, 3, 3], 96, 4, [1, 1], [1, 1], [1, 1])
        with pytest.raises(ValueError):
            torch.ops.quanto.qbytes_conv2d(x.float(), w, s, None, [1, 1], [1, 1], [1, 1])
