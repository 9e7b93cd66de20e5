"""CPU: the HQQ restatement (oracle/hqq_oracle.py) and the package's HqqOptimizer composition against the reference
(tests/golden/hqq.npz, written by oracle/gen_golden_hqq.py), QLinear freezing through the composition, the export."""
import os

import numpy as np
import pytest
import torch

import quanto_b200 as q
from oracle import hqq_oracle as H
from oracle import quanto_oracle as O

TORCH_DT = {"bf16": torch.bfloat16, "f16": torch.float16}
ALL = np.arange(65536, dtype=np.uint32).astype(np.uint16)


@pytest.fixture(scope="module")
def z(golden_dir):
    return np.load(os.path.join(golden_dir, "hqq.npz"))


def _bits_equal(a, b, tag):
    a = np.asarray(a, np.uint16)
    b = np.asarray(b, np.uint16)
    inf = 0x7F80 if tag == "bf16" else 0x7C00
    nan_a, nan_b = (a & 0x7FFF) > inf, (b & 0x7FFF) > inf
    return bool(np.array_equal(nan_a, nan_b) and np.array_equal(a[~nan_a], b[~nan_b]))


def cases(z):
    for i in range(int(z["n_hqq"])):
        p = f"h{i}_"
        tag = str(z[p + "tag"])
        N, K, G = (int(v) for v in z[p + "shape"])
        lp, beta, kappa, iters = (float(v) for v in z[p + "params"])
        yield i, p, tag, N, K, G, dict(lp_norm=lp, beta=beta, kappa=kappa, iters=int(iters))


@pytest.mark.parametrize("tag", ["bf16", "f16"])
def test_pow_matches_reference_on_every_pattern(z, tag):
    a = np.abs(O.to_f32(ALL, tag))
    assert _bits_equal(O.from_f32(H.lp_pow(a, 0.7, tag), tag), z[f"pow_{tag}"], tag)


@pytest.mark.parametrize("tag", ["bf16", "f16"])
def test_shrink_matches_reference(z, tag):
    j = 0
    while f"shrink_{tag}_{j}_out" in z:
        p = f"shrink_{tag}_{j}_"
        x = z[p + "x"] if p + "x" in z else ALL
        out = H.shrink_lp(O.to_f32(x, tag), tag, float(z[p + "beta"]), float(z[p + "lp"]))
        assert _bits_equal(O.from_f32(out, tag), z[p + "out"], tag), (tag, j)
        j += 1
    assert j == 6


def test_oracle_matches_reference_hqq(z):
    stops = set()
    for i, p, tag, N, K, G, kw in cases(z):
        bits = int(z[p + "bits"])
        zp = bool(z[p + "zeropoint"])
        w = O.to_f32(z[p + "W"], tag).reshape(-1, G)
        scale, shift, errors, accepted = H.hqq(w, tag, bits, zeropoint=zp, **kw)
        assert np.array_equal(scale.reshape(-1), z[p + "scale"].reshape(-1)), i
        assert np.array_equal(shift.reshape(-1), z[p + "shift"].reshape(-1)), i
        assert errors == list(z[p + "errors"]), (i, errors, list(z[p + "errors"]))
        stops.add(accepted)
    assert 0 in stops and len(stops) > 2, stops  # some case stops at the first iteration, others later


def _composition(w_bits, tag, bits, G, zp, kw):
    W = torch.from_numpy(w_bits.view(np.int16)).view(TORCH_DT[tag])
    qt = q.qint4 if bits == 4 else q.qint2
    return q.HqqOptimizer(**kw)(W, qtype=qt, axis=0, group_size=G, zeropoint=zp)


def _bits(t):
    t = t.contiguous()
    return t.numpy() if t.dtype == torch.uint8 else t.view(torch.int16).numpy().view(np.uint16)


def test_composition_on_cpu_matches_reference(z):
    for i, p, tag, N, K, G, kw in cases(z):
        W = z[p + "W"].reshape(N, K)
        scale, shift = _composition(W, tag, int(z[p + "bits"]), G, bool(z[p + "zeropoint"]), kw)
        assert np.array_equal(_bits(scale).reshape(-1), z[p + "scale"].reshape(-1)), i
        assert np.array_equal(_bits(shift).reshape(-1), z[p + "shift"].reshape(-1)), i


def test_verbose_prints_the_errors(z, capsys):
    i, p, tag, N, K, G, kw = next(cases(z))
    _composition(z[p + "W"].reshape(N, K), tag, int(z[p + "bits"]), G, False, dict(kw, verbose=True))
    lines = capsys.readouterr().out.splitlines()
    errors = list(z[p + "errors"])
    assert lines[0] == f"Start error: {errors[0]:.6f}"
    assert lines[1:] == [f"HQQ error at it #{k}: {e:.6f}" for k, e in enumerate(errors[1:])]


def test_qlinear_freeze_on_cpu_matches_reference(z):
    W = torch.from_numpy(z["qlinear_W"].view(np.int16)).view(torch.bfloat16)
    lin = torch.nn.Linear(W.shape[1], W.shape[0], bias=False).to(torch.bfloat16)
    with torch.no_grad():
        lin.weight.copy_(W)
    ql = q.QLinear.from_module(lin, weights=q.qint4, optimizer=q.HqqOptimizer())
    ql.freeze()
    assert ql.weight_group_size == int(z["qlinear_group"])
    assert np.array_equal(ql.weight._data._data.numpy(), z["qlinear_packed"])
    assert np.array_equal(_bits(ql.weight._scale).reshape(-1), z["qlinear_scale"].reshape(-1))
    assert np.array_equal(_bits(ql.weight._shift).reshape(-1), z["qlinear_shift"].reshape(-1))


def test_exports():
    from quanto_b200.tensor import HqqOptimizer

    assert q.HqqOptimizer is HqqOptimizer
    opt = HqqOptimizer()
    assert (opt.lp_norm, opt.beta, opt.kappa, opt.iters, opt.verbose) == (0.7, 1e1, 1.01, 20, False)
    assert isinstance(opt, q.MaxOptimizer)
