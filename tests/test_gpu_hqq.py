"""GPU parity of the fused HQQ freeze (csrc/hqq.cu) against the oracle (oracle/hqq_oracle.py) and the fixture written
from the real reference (tests/golden/hqq.npz, oracle/gen_golden_hqq.py).  Scale, shift, zero-points, packed bytes, the
per-iteration errors and the stop index are integer / bit-pattern results: the bar is bit-exact."""
import os

import numpy as np
import pytest
import torch

import quanto_b200 as q
from helpers import O, bits_to_torch, torch_to_bits, torch_to_f32
from oracle import hqq_oracle as H
from quanto_b200 import _native

pytestmark = pytest.mark.gpu
TDT = {"f16": torch.float16, "bf16": torch.bfloat16}
QT = {2: q.qint2, 4: q.qint4}
ALL = np.arange(65536, dtype=np.uint32).astype(np.uint16)
DEFAULTS = dict(lp_norm=0.7, beta=10.0, kappa=1.01, iters=20)


@pytest.fixture(scope="module")
def z(golden_dir):
    return np.load(os.path.join(golden_dir, "hqq.npz"))


def _bits_equal(a, b, tag):
    a, b = np.asarray(a, np.uint16), np.asarray(b, np.uint16)
    inf = 0x7F80 if tag == "bf16" else 0x7C00
    nan_a, nan_b = (a & 0x7FFF) > inf, (b & 0x7FFF) > inf
    return bool(np.array_equal(nan_a, nan_b) and np.array_equal(a[~nan_a], b[~nan_b]))


def _weight(n, k, tag, seed, spread=0.02):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, k, generator=g) * spread).to(TDT[tag])


def _op(w, bits, G, zeropoint=False, **kw):
    p = dict(DEFAULTS, **kw)
    return torch.ops.quanto.quantize_qbits_hqq(w.cuda(), bits, G, zeropoint, p["lp_norm"], p["beta"], p["kappa"],
                                               p["iters"])


def _check_against_oracle(w, tag, bits, G, zeropoint=False, rows=None, **kw):
    """Run the op on w [N, K] and compare everything with the oracle; `rows` restricts the row-wise outputs to a band
    (the errors and the stop index always cover the whole weight).  Returns the accepted count."""
    p = dict(DEFAULTS, **kw)
    packed, scale, shift, errors = _op(w, bits, G, zeropoint, **kw)
    wg = torch_to_f32(w).reshape(-1, G)
    s_ref, z_ref, e_ref, acc = H.hqq(wg, tag, bits, zeropoint=zeropoint, trajectory=True, **p)
    errors = errors.cpu().numpy()
    assert list(errors[: p["iters"] + 1].astype(np.float64)) == e_ref, (errors, e_ref)
    assert int(errors[p["iters"] + 1]) == acc
    sel = slice(None) if rows is None else rows
    assert np.array_equal(torch_to_bits(scale).reshape(-1)[sel], s_ref.reshape(-1)[sel])
    got_shift = shift.cpu().numpy() if zeropoint else torch_to_bits(shift)
    assert np.array_equal(got_shift.reshape(-1)[sel], z_ref.reshape(-1)[sel])
    packed_ref = H.quantize_packed(wg, tag, bits, s_ref, z_ref, zeropoint)
    if rows is None:
        assert np.array_equal(packed.cpu().numpy(), packed_ref)
    else:
        assert np.array_equal(packed.cpu().numpy()[sel], packed_ref[sel])
    return acc


# ------------------------------------------------------------------------------------------------------ shrink
@pytest.mark.parametrize("tag", ["bf16", "f16"])
def test_shrink_every_pattern_matches_fixture(z, tag):
    x = bits_to_torch(ALL, tag)
    out = torch.ops.quanto.hqq_shrink(x, 10.0, 0.7)
    assert _bits_equal(torch_to_bits(out), z[f"shrink_{tag}_0_out"], tag)
    for j in range(1, 6):
        p = f"shrink_{tag}_{j}_"
        out = torch.ops.quanto.hqq_shrink(bits_to_torch(z[p + "x"], tag), float(z[p + "beta"]), float(z[p + "lp"]))
        assert _bits_equal(torch_to_bits(out), z[p + "out"], tag), j


@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("lp, beta", [(1.0, 10.0), (1.0, 13.7), (0.7, 10.0 * 1.01 ** 19), (0.5, 3.0), (2.0, 7.0)])
def test_shrink_every_pattern_matches_oracle(tag, lp, beta):
    out = torch.ops.quanto.hqq_shrink(bits_to_torch(ALL, tag), beta, lp)
    ref = O.from_f32(H.shrink_lp(O.to_f32(ALL, tag), tag, beta, lp), tag)
    assert _bits_equal(torch_to_bits(out), ref, tag)


# -------------------------------------------------------------------------------------------- fixture replay
def _cases(z):
    for i in range(int(z["n_hqq"])):
        p = f"h{i}_"
        N, K, G = (int(v) for v in z[p + "shape"])
        lp, beta, kappa, iters = (float(v) for v in z[p + "params"])
        yield (p, str(z[p + "tag"]), int(z[p + "bits"]), N, K, G, bool(z[p + "zeropoint"]),
               dict(lp_norm=lp, beta=beta, kappa=kappa, iters=int(iters)))


def _reference_accepted(errors, iters):
    """The accepted count the reference's loop reached, from its recorded errors (start, then one per iteration)."""
    n = len(errors) - 1
    if iters == 0:
        return 0
    return n if n == iters and (n == 0 or errors[-1] < min(errors[:-1])) else n - 1


def test_fixture_replay_through_the_op(z):
    for p, tag, bits, N, K, G, zp, kw in _cases(z):
        w = bits_to_torch(z[p + "W"], tag).reshape(N, K)
        packed, scale, shift, errors = _op(w, bits, G, zp, **kw)
        assert np.array_equal(torch_to_bits(scale).reshape(-1), z[p + "scale"].reshape(-1)), p
        got = shift.cpu().numpy() if zp else torch_to_bits(shift)
        assert np.array_equal(got.reshape(-1), z[p + "shift"].reshape(-1)), p
        ref_errors = list(z[p + "errors"])
        errors = errors.cpu().numpy().astype(np.float64)
        assert list(errors[: len(ref_errors)]) == ref_errors, p
        assert int(errors[kw["iters"] + 1]) == _reference_accepted(ref_errors, kw["iters"]), p
        wg = torch_to_f32(w).reshape(-1, G)
        assert np.array_equal(packed.cpu().numpy(), H.quantize_packed(wg, tag, bits, z[p + "scale"], z[p + "shift"], zp))


def _freeze(w, qt, G, optimizer):
    lin = torch.nn.Linear(w.shape[1], w.shape[0], bias=False).to(w.dtype)
    with torch.no_grad():
        lin.weight.copy_(w.cpu())
    ql = q.QLinear.from_module(lin.cuda(), weights=qt, optimizer=optimizer)
    assert ql.weight.is_cuda
    ql.weight_group_size = G
    ql.freeze()
    return ql


def test_fixture_replay_through_qlinear_freeze(z):
    for p, tag, bits, N, K, G, zp, kw in _cases(z):
        if zp:
            continue  # QLinear stores float shifts
        ql = _freeze(bits_to_torch(z[p + "W"], tag).reshape(N, K), QT[bits], G, q.HqqOptimizer(**kw))
        wq = ql.weight
        assert np.array_equal(torch_to_bits(wq._scale).reshape(-1), z[p + "scale"].reshape(-1)), p
        assert np.array_equal(torch_to_bits(wq._shift).reshape(-1), z[p + "shift"].reshape(-1)), p
        wg = O.to_f32(z[p + "W"], tag).reshape(-1, G)
        packed_ref = H.quantize_packed(wg, tag, bits, z[p + "scale"], z[p + "shift"], False)
        assert np.array_equal(wq._data._data.cpu().numpy(), packed_ref), p
    w = bits_to_torch(z["qlinear_W"], "bf16")
    ql = _freeze(w, q.qint4, int(z["qlinear_group"]), q.HqqOptimizer())
    assert np.array_equal(ql.weight._data._data.cpu().numpy(), z["qlinear_packed"])
    assert np.array_equal(torch_to_bits(ql.weight._scale).reshape(-1), z["qlinear_scale"].reshape(-1))
    assert np.array_equal(torch_to_bits(ql.weight._shift).reshape(-1), z["qlinear_shift"].reshape(-1))


# ----------------------------------------------------------------------------------------- full-size weights
def test_full_oracle_4096_square():
    acc = _check_against_oracle(_weight(4096, 4096, "bf16", 1), "bf16", 4, 128)
    assert acc > 0


@pytest.mark.parametrize("N, K", [(14336, 4096), (4096, 14336)])
def test_llama_ffn_band_and_stop_index(N, K):
    """Rows are independent once the stop index is fixed: a band of rows is checked byte for byte, the errors and the
    stop index over the whole weight (6 iterations keep the oracle's time in bounds; the stop comes earlier)."""
    G = 128
    rows = N * K // G
    acc = _check_against_oracle(_weight(N, K, "bf16", 2), "bf16", 4, G, rows=slice(rows // 2 - 4096, rows // 2 + 4096),
                                iters=6)
    assert 0 < acc < 6


# ----------------------------------------------------------------------------------------------------- edges
@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("bits, N, K, G", [(4, 24, 384, 96), (4, 12, 384, 192), (4, 10, 512, 256), (2, 40, 256, 256),
                                           (2, 7, 384, 192), (4, 9, 96, 32), (2, 33, 64, 8), (4, 3, 256, 64)])
def test_group_sizes_and_odd_rows(tag, bits, N, K, G):
    _check_against_oracle(_weight(N, K, tag, N + K + G), tag, bits, G)


@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("bits", [2, 4])
def test_zeropoint_and_constant_groups(tag, bits):
    w = _weight(30, 256, tag, 5).float()
    wg = w.view(-1, 64)
    wg[2::7] = 0.0
    wg[5::9] = -0.0078125
    _check_against_oracle(w.to(TDT[tag]), tag, bits, 64, zeropoint=True)
    _check_against_oracle(w.to(TDT[tag]), tag, bits, 64)


@pytest.mark.parametrize("kw", [dict(iters=0), dict(iters=1), dict(lp_norm=1.0), dict(lp_norm=1.0, beta=3.0, kappa=1.3),
                                dict(lp_norm=0.5, beta=40.0, iters=64), dict(lp_norm=2.0, kappa=1.0)])
def test_parameters(kw):
    _check_against_oracle(_weight(64, 512, "bf16", 7), "bf16", 4, 128, **kw)
    _check_against_oracle(_weight(48, 384, "f16", 8), "f16", 2, 64, **kw)


def test_stop_at_the_first_iteration():
    """A weight whose groups already sit on the quantization grid: the first HQQ step cannot improve on the start."""
    g = torch.Generator().manual_seed(11)
    codes = torch.randint(0, 16, (32, 256), generator=g).float()
    codes[:, 0::64], codes[:, 1::64] = 0.0, 15.0  # every group spans the full code range
    w = (codes * 2.0 ** -7 - 0.0625).to(torch.bfloat16)
    assert _check_against_oracle(w, "bf16", 4, 64) == 0


def test_two_launches_give_identical_bytes():
    w = _weight(4096, 4096, "f16", 3).cuda()
    a = _op(w, 4, 128)
    b = _op(w, 4, 128)
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.uint8) if x.dtype != torch.float32 else x, y.view(torch.uint8)
                           if y.dtype != torch.float32 else y)


# -------------------------------------------------------------------------------- declined -> composition
def test_declined_inputs_run_the_composition():
    w32 = _weight(64, 256, "bf16", 4).float().cuda()
    with pytest.raises(_native.UnsupportedConfiguration):
        _op(w32, 4, 128)
    opt = q.HqqOptimizer()
    scale, shift = opt(w32, q.qint4, axis=0, group_size=128)
    s_ref, z_ref = opt.optimize(q.tensor.grouped.group(w32, 0, 128), q.qint4, 0)
    assert torch.equal(scale, s_ref) and torch.equal(shift, z_ref)
    w = _weight(64, 512, "bf16", 4).cuda()
    assert opt.fused(w, q.qint4, -1, 32) is None
    scale, shift = opt(w, q.qint4, axis=-1, group_size=32)
    s_ref, z_ref = opt.optimize(q.tensor.grouped.group(w, -1, 32), q.qint4, -1)
    assert torch.equal(scale, s_ref) and torch.equal(shift, z_ref)
    with pytest.raises(_native.UnsupportedConfiguration):
        _op(w, 4, 512)  # a per-axis row longer than 256
    assert opt.fused(w, q.qint4, 0, None) is None
    scale, shift = opt(w, q.qint4, axis=0)
    assert scale.shape == (64, 1)
    with pytest.raises(_native.UnsupportedConfiguration):
        _op(w, 4, 128, iters=65)
    with pytest.raises(_native.UnsupportedConfiguration):
        _op(w, 4, 128, lp_norm=4.0)


# ------------------------------------------------------------------------------------- frozen layer, quality
def test_frozen_hqq_layer_forward_and_state_dict():
    w = _weight(256, 512, "bf16", 9)
    ql_hqq = _freeze(w, q.qint4, 128, q.HqqOptimizer())
    ql_max = _freeze(w, q.qint4, 128, q.MaxOptimizer())
    assert set(ql_hqq.state_dict()) == set(ql_max.state_dict())
    wq = ql_hqq.weight
    x = torch.randn(16, 512, generator=torch.Generator().manual_seed(1)).to(torch.bfloat16).cuda()
    with torch.no_grad():
        y = ql_hqq(x)
    y_ref = torch.ops.quanto.qbits_mm(x, wq._data._data, wq._scale, wq._shift, None, 256, 128, 4)
    assert torch.equal(y, y_ref)
    deq = O.dequantize_qbits(wq._data._data.cpu().numpy(), 4, torch_to_bits(wq._scale), torch_to_bits(wq._shift),
                             "bf16", 256, 512, 128)
    y64, _, tol = O.linear_from_dequantized(torch_to_f32(x), O.to_f32(deq, "bf16"), None, "bf16")
    bound = 1.02 * tol + O.accumulate_allowance(torch_to_f32(x), O.to_f32(deq, "bf16"))
    assert np.all(np.abs(y.float().cpu().numpy().astype(np.float64) - y64) <= bound)


@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("bits", [2, 4])
def test_quality_not_worse_than_max(tag, bits):
    """The reference test's property: the mean absolute error with the HQQ shift is at most MaxOptimizer's."""
    w = _weight(1024, 1024, tag, 12).cuda()
    qt = QT[bits]

    def mean_error(opt):
        scale, shift = opt(w, qt, axis=0, group_size=64)
        wq = q.quantize_weight(w, qtype=qt, axis=0, scale=scale, shift=shift, group_size=64)
        return torch.abs(w - wq.dequantize()).mean()

    assert mean_error(q.HqqOptimizer()) <= mean_error(q.MaxOptimizer())
