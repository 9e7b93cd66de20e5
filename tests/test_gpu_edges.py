"""Edges of the shipped kernels that the shape-by-shape suites do not reach.

* float8_e4m3fnuz end to end: the quantize_symmetric encoder, the staging-warp decoder of the weight-only wgmma kernel,
  the CUDA-core decoder, and QLinear layers, against the oracle and fixtures of the real reference (tests/golden/fnuz.npz).
* An instantiation census: one row per shipped gemm_tc_kernel instantiation, each forced by the test overrides and run at
  one shape that is one row past a tile boundary, ragged in N and has a K tail (the zero-filled 16-byte chunks of the
  staging loops).
* Many tiles per CTA with fewer k-blocks than pipeline stages: the staging groups start tiles ahead of the consumers.
* int4 group sizes that are multiples of 64 but not powers of two (the division path of the staging warps and gemvs).
* NaN weight codes: the reference computes W.to(dtype) * scale and a matmul, so one NaN weight is one NaN column.
"""
import contextlib
import os

import numpy as np
import pytest
import torch

import quanto_b200 as q
from helpers import (O, band_rows, bits_to_torch, cabi_dequantize_qbits, cabi_qbits_mm, cabi_qbytes_mm,
                     cabi_quantize_symmetric, check_full_against_device_fp32, check_linear, make_qbits_weights, native,
                     torch_to_bits, torch_to_f32)

pytestmark = pytest.mark.gpu
FNUZ = torch.float8_e4m3fnuz
TDT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16}


def _fnuz_golden(golden_dir):
    return np.load(os.path.join(golden_dir, "fnuz.npz"))


def _overrides(pairs):
    """Nested qb200_test_override contexts for (key name, value) pairs."""
    n = native()
    stack = contextlib.ExitStack()
    for key, value in pairs:
        stack.enter_context(n.test_override(getattr(n, key), value))
    return stack


def _check_weight_only(y, a, w, s, bias, tag, label):
    """Weight-only 8-bit bound of test_qbytes_mm_weight_only_tensor_path: operands rnd(A), rnd(scale * W) exactly as the
    reference's python path forms them, only the fp32 summation order free."""
    ap, wp = O.qbytes_mm_operands(a, w, s, tag)
    y64, _, tol = O.linear_from_dequantized(ap, wp, bias, tag)
    bound = 1.02 * tol + O.accumulate_allowance(ap, wp)
    err = np.abs(torch_to_f32(y).astype(np.float64) - y64)
    assert np.all(err <= bound), (label, float(np.max(err / bound)), np.unravel_index(np.argmax(err / bound), err.shape))


def _check_fp8_native(y, a_bits, akind, w_bits, wkind, s, tag, label):
    """The bound of test_qbytes_mm_fp8_native: exact products, fp32 sum, scale applied to the fp32 result."""
    y64, _ = O.qbytes_mm_fp8_native(a_bits, akind, w_bits, wkind, s, tag)
    a, w = O.fp8_bits_to_f32(a_bits, akind), O.fp8_bits_to_f32(w_bits, wkind)
    bound = 0.51 * O.ulp(y64, tag) + O.accumulate_allowance(a, w) * np.abs(s).reshape(1, -1)
    err = np.abs(torch_to_f32(y).astype(np.float64) - y64)
    assert np.all(err <= bound), (label, float(np.max(err / bound)), np.unravel_index(np.argmax(err / bound), err.shape))


def _fp8_codes(kind, shape, rng, spread=3.0):
    """Random finite fp8 codes of `kind` (values clipped to a range every format represents)."""
    return O.f32_to_fp8_bits(np.clip(rng.standard_normal(shape, dtype=np.float32) * spread, -200, 200), kind)


def _fnuz_all_codes(N, K, rng):
    """[N, K] e4m3fnuz codes containing every one of the 255 non-NaN codes (N * K >= 255), shuffled."""
    codes = np.array([c for c in range(256) if c != 0x80], np.uint8)
    return rng.permutation(np.resize(codes, N * K)).reshape(N, K)


# --------------------------------------------------------------------------------- e4m3fnuz: quantize_symmetric
def test_fnuz_quantize_symmetric_golden(golden_dir):
    z = _fnuz_golden(golden_dir)
    for i in range(int(z["n_quantize"])):
        p = f"q{i}_"
        in_tag, axis = str(z[p + "in_tag"]), int(z[p + "axis"])
        axis = None if axis == -2 else axis
        base = bits_to_torch(z[p + "base"], in_tag)
        scale = bits_to_torch(z[p + "scale"], in_tag).reshape(z[p + "scale"].shape)
        out = cabi_quantize_symmetric(base, FNUZ, axis, scale)
        assert np.array_equal(torch_to_bits(out), z[p + "out"]), (i, in_tag, axis)
        op = torch.ops.quanto.quantize_symmetric(base, dtype=FNUZ, axis=axis, scale=scale)  # the reference-facing op
        assert op.dtype == FNUZ and np.array_equal(torch_to_bits(op), z[p + "out"]), (i, in_tag, axis)


@pytest.mark.parametrize("in_tag", ["f32", "f16", "bf16"])
@pytest.mark.parametrize("axis", [None, 0, -1])
def test_fnuz_quantize_symmetric_large(in_tag, axis):
    rng = np.random.default_rng(13)
    base = rng.standard_normal((1024, 2048), dtype=np.float32) * 2
    base[:, :16] *= 1e-6  # quotients far below the smallest subnormal, both signs: 0x00, never 0x80
    base[7] = 0.0         # an all-zero row: per-row scale 0, quotient 0/0 -> NaN -> 0x80
    base = O.round_to(base, in_tag)
    if axis is None:
        scale = O.round_to(np.array(np.abs(base).max() / 300, np.float32), in_tag)  # quotients past +-240 saturate
    elif axis == 0:
        scale = O.round_to(np.abs(base).max(axis=1, keepdims=True) / 250, in_tag)
    else:
        scale = O.round_to(np.abs(base).max(axis=0, keepdims=True) / 250, in_tag)
    ref = O.quantize_symmetric(base, in_tag, "e4m3fnuz", scale)
    assert np.sum((ref & 0x7F) == 0x7F) > 0 and np.sum((ref == 0) & np.signbit(base)) > 0
    assert axis != 0 or np.any(ref == 0x80)
    out = cabi_quantize_symmetric(bits_to_torch(O.from_f32(base, in_tag), in_tag), FNUZ, axis,
                                  bits_to_torch(O.from_f32(scale, in_tag), in_tag))
    got = torch_to_bits(out)
    assert np.array_equal(got, ref), int(np.sum(got != ref))


def test_fnuz_quantize_symmetric_bf16_all_values():
    """Every finite bf16 value against 48 scales and scale 0 (x / 0 = +-inf saturates, 0 / 0 = NaN -> 0x80)."""
    bits = np.arange(65536, dtype=np.uint16)
    bits = bits[np.isfinite(O.bf16_bits_to_f32(bits))]
    bits = np.resize(bits, (255, 256))
    base = O.bf16_bits_to_f32(bits)
    rng = np.random.default_rng(5)
    scales = np.concatenate([O.round_to(np.exp(rng.uniform(-12, 6, 40)).astype(np.float32), "bf16"),
                             np.array([1.0, 0.5, 3.0, 0.0078125, 1.1754944e-38, 3.0e38, 7.0, 0.33203125, 0.0], np.float32)])
    for sc in scales:
        sc = O.round_to(np.array(sc, np.float32), "bf16")
        ref = O.quantize_symmetric(base, "bf16", "e4m3fnuz", sc)
        out = cabi_quantize_symmetric(bits_to_torch(bits, "bf16"), FNUZ, None, bits_to_torch(O.from_f32(sc, "bf16"), "bf16"))
        got = torch_to_bits(out)
        assert np.array_equal(got, ref), (float(sc), int(np.sum(got != ref)))


# --------------------------------------------------------------------------------- e4m3fnuz: qbytes_mm / QLinear
@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("tile_m", [64, 128])
def test_fnuz_weights_tensor_path(tag, tile_m):
    """Weight-only wgmma kernel, both tile heights, with every non-NaN e4m3fnuz code in the weights."""
    M, N, K = 200, 300, 528
    rng = np.random.default_rng(21)
    a = O.round_to(rng.standard_normal((M, K), dtype=np.float32), tag)
    w_bits = _fnuz_all_codes(N, K, rng)
    s = O.round_to(rng.random(N, dtype=np.float32) / 1e2 + 1e-4, tag)
    bias = O.round_to(rng.standard_normal(N, dtype=np.float32), tag)
    with _overrides([("OVR_TILE_M", tile_m)]):
        y, family = cabi_qbytes_mm(bits_to_torch(O.from_f32(a, tag), tag), bits_to_torch(w_bits, "e4m3fnuz"),
                                   bits_to_torch(O.from_f32(s, tag), tag), bits_to_torch(O.from_f32(bias, tag), tag))
        torch.cuda.synchronize()
    assert family == 1
    _check_weight_only(y, a, O.fp8_bits_to_f32(w_bits, "e4m3fnuz"), s, bias, tag, (tag, tile_m))


@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("akind", ["f32", "int8", "e4m3fnuz"])
def test_fnuz_weights_cuda_core_route(tag, akind):
    """Activations the tensor-core kernels do not take run on the CUDA-core kernel and its e4m3fnuz decoder."""
    M, N, K = 33, 300, 96
    rng = np.random.default_rng(22)
    if akind == "f32":
        a_store = rng.standard_normal((M, K), dtype=np.float32)
        a = a_store
    elif akind == "int8":
        a_store = rng.integers(-128, 128, size=(M, K), dtype=np.int8)
        a = a_store.astype(np.float32)
    else:
        a_store = _fnuz_all_codes(M, K, rng)
        a = O.fp8_bits_to_f32(a_store, "e4m3fnuz")
    w_bits = _fnuz_all_codes(N, K, rng)
    s = O.round_to(rng.random(N, dtype=np.float32) / 1e3 + 1e-5, tag)
    y, family = cabi_qbytes_mm(bits_to_torch(a_store, akind), bits_to_torch(w_bits, "e4m3fnuz"),
                               bits_to_torch(O.from_f32(s, tag), tag))
    torch.cuda.synchronize()
    assert family == 2
    _check_weight_only(y, a, O.fp8_bits_to_f32(w_bits, "e4m3fnuz"), s, None, tag, (tag, akind))


def test_fnuz_qbytes_mm_golden(golden_dir):
    """The reference's own qbytes_mm outputs with e4m3fnuz weights (K = 32, 50, 64, 80; fp16 / bf16 / f32 / int8 / e4m3fnuz
    activations)."""
    z = _fnuz_golden(golden_dir)
    for i in range(int(z["n_mm"])):
        p = f"m{i}_"
        akind, tag = str(z[p + "akind"]), str(z[p + "tag"])
        A = bits_to_torch(z[p + "A"], tag if akind == "same" else akind)
        y, family = cabi_qbytes_mm(A, bits_to_torch(z[p + "W"], "e4m3fnuz"), bits_to_torch(z[p + "scales"], tag).reshape(-1))
        torch.cuda.synchronize()
        K = z[p + "A"].shape[1]
        assert family == (1 if akind == "same" and K % 16 == 0 else 2), (i, akind, K, family)
        a = O.to_f32(z[p + "A"], tag if akind == "same" else akind) if akind != "int8" else z[p + "A"].astype(np.float32)
        _check_weight_only(y, a, O.fp8_bits_to_f32(z[p + "W"], "e4m3fnuz"), O.to_f32(z[p + "scales"], tag), None, tag,
                           (i, akind, tag))
        yref = O.to_f32(z[p + "y"], tag).astype(np.float64)
        rel = np.linalg.norm(torch_to_f32(y) - yref) / np.linalg.norm(yref)
        assert rel < 1e-3, (i, rel)


def _tt(arr, dtype):
    if dtype in (torch.float16, torch.bfloat16):
        return torch.from_numpy(arr.view(np.int16).copy()).view(dtype)
    return torch.from_numpy(arr.copy())


def test_fnuz_qlinear_golden(golden_dir):
    """QLinear(weights=qfloat8_e4m3fnuz) and QLinear(activations=qfloat8_e4m3fnuz) loaded from the reference's state dict,
    with the tolerances of test_qlinear_matches_reference_outputs."""
    z = _fnuz_golden(golden_dir)
    for i in range(int(z["n_qlinear"])):
        p = f"l{i}_"
        tag = str(z[p + "tag"])
        dtype = TDT[tag]
        N, K, M, _ = (int(v) for v in z[p + "shape"])
        wq = q.qtypes[str(z[p + "wq"])]
        aq = None if str(z[p + "aq"]) == "none" else q.qtypes[str(z[p + "aq"])]
        lin = torch.nn.Linear(K, N, bias=True).to(dtype)
        ql = q.QLinear.from_module(lin, weights=wq, activations=aq)
        sd = {"bias": _tt(z[p + "bias"], dtype), "input_scale": _tt(z[p + "input_scale"], dtype).reshape(()),
              "output_scale": _tt(z[p + "output_scale"], dtype).reshape(())}
        for key in z.files:
            if key.startswith(p + "sd_"):
                name, arr = key[len(p) + 3:], z[key]
                if name.endswith("_data") and wq.is_floating_point:
                    sd[name] = torch.from_numpy(arr.copy()).view(wq.dtype)
                elif name.endswith("_data"):
                    sd[name] = torch.from_numpy(arr.copy())
                else:
                    sd[name] = _tt(arr, dtype)
        ql.load_state_dict(sd)
        ql = ql.cuda()
        with torch.no_grad():
            y = ql(_tt(z[p + "x"], dtype).cuda())
        torch.cuda.synchronize()
        if aq is None:
            yref = O.to_f32(z[p + "y"], tag).astype(np.float64)
            rel = np.linalg.norm(torch_to_f32(y).astype(np.float64) - yref) / np.linalg.norm(yref)
            assert rel < 1e-3, (i, rel)
        else:
            assert isinstance(y, q.ActivationQBytesTensor) and y._data.dtype == FNUZ
            mismatch = np.mean(torch_to_bits(y._data) != z[p + "y_data"])
            assert mismatch < 0.05, (i, mismatch)


# --------------------------------------------------------------------------------- instantiation census
# One row per shipped gemm_tc_kernel instantiation (36): (id, family, variant, tile M, tile N, M, N, K, output tag).
# M is one row past a tile boundary, N is ragged, K has a tail: K % 64 in {16, 32, 48} for the staged 8-bit paths,
# K % 128 != 0 for int8 x int8 (TMA), K % 64 == 32 with groups of 32 for int4.
def _census():
    rows = []
    # api_qbits.cu GemmCfg<KIND, BSrc::INT4, MWG, 128, WT, ZP>: bf16/f16 x float shift / zero-point, MWG 1 / 2
    for tag in ("bf16", "f16"):
        for zp in (False, True):
            for tm in (64, 128):
                rows.append((f"int4-{tag}-{'zp' if zp else 'shift'}-m{tm}", "int4", zp, tm, 128,
                             65 if tm == 64 else 129, 336, 352, tag))
    # api_qbytes.cu GemmCfg<MmaKind::I8, BSrc::TMA, MWG, BN>
    for j, (tm, bn) in enumerate(((64, 128), (64, 256), (128, 128), (128, 256))):
        rows.append((f"int8-m{tm}-n{bn}", "int8", None, tm, bn, 65 if tm == 64 else 200, 301, 592,
                     ("bf16", "f16", "f32", "bf16")[j]))
    # api_qbytes.cu F8Cfg<MWG, WKIND, AKIND>: (activation, weight) pairs, MWG 1 / 2
    for j, (ak, wk) in enumerate((("e4m3fn", "e4m3fn"), ("e5m2", "e4m3fn"), ("e4m3fn", "e5m2"), ("e5m2", "e5m2"))):
        for tm in (64, 128):
            rows.append((f"fp8-{ak}-{wk}-m{tm}", "fp8", (ak, wk), tm, 128, 65 if tm == 64 else 129, 301,
                         (528, 544, 560)[(2 * j + tm // 128) % 3], ("bf16", "f16")[j % 2]))
    # api_qbytes.cu GemmCfg<KIND, BSrc::BYTES, MWG, 128, WT, false, WKIND>: bf16/f16 activations x
    # int8/e4m3fn/e5m2/e4m3fnuz weights, MWG 2 / 1
    for tag in ("bf16", "f16"):
        for j, wk in enumerate(("int8", "e4m3fn", "e5m2", "e4m3fnuz")):
            for tm in (64, 128):
                rows.append((f"w8-{tag}-{wk}-m{tm}", "w8", wk, tm, 128, 65 if tm == 64 else 200, 301,
                             (528, 544, 560)[(j + tm // 128) % 3], tag))
    return rows


CENSUS = _census()
assert len(CENSUS) == 36 and len({r[0] for r in CENSUS}) == 36


@pytest.mark.parametrize("row", CENSUS, ids=[r[0] for r in CENSUS])
def test_instantiation_census(row):
    name, fam, var, tm, bn, M, N, K, tag = row
    rng = np.random.default_rng(len(name) * 1000 + M + N + K)
    ovr = [("OVR_TILE_M", tm)] + ([("OVR_QBYTES_TILE_N", bn)] if fam == "int8" else [])
    bias = O.round_to(rng.standard_normal(N, dtype=np.float32), tag) if M % 2 else None
    bias_t = None if bias is None else bits_to_torch(O.from_f32(bias, tag), tag)
    lib = native().load()
    if fam == "int4":
        G, zp = 32, var
        assert K % 64 == 32 and (N // 2) % 64 != 0
        _, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=M + K, zeropoint=zp)
        x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
        deq_bits = O.dequantize_qbits(packed, 4, scale, shift, tag, N, K, G, shift_is_int=zp)
        shift_t = torch.from_numpy(shift).cuda() if zp else bits_to_torch(shift, tag)
        bias_bits = None if bias is None else O.from_f32(bias, tag)
        with _overrides(ovr):
            y = cabi_qbits_mm(bits_to_torch(x_bits, tag), torch.from_numpy(packed).cuda(), bits_to_torch(scale, tag),
                              shift_t, bias_t, N, K, G)
            family = lib.qb200_last_kernel_family()
            torch.cuda.synchronize()
        assert family == 1, name
        check_linear(y, x_bits, deq_bits, bias_bits, tag, name)
        return
    assert N % 2 == 1 and N % 128 != 0
    if fam == "int8":
        assert K % 128 != 0
        A = rng.integers(-128, 128, size=(M, K), dtype=np.int8)
        W = rng.integers(-128, 128, size=(N, K), dtype=np.int8)
        s = O.round_to(rng.random(N, dtype=np.float32) / 1e3 + 1e-5, tag)
        with _overrides(ovr):
            y, family = cabi_qbytes_mm(torch.from_numpy(A).cuda(), torch.from_numpy(W).cuda(),
                                       bits_to_torch(O.from_f32(s, tag), tag), bias_t)
            torch.cuda.synchronize()
        assert family == 1, name
        ref = O.to_f32(O.qbytes_int_mm(A, W, s, tag), tag)
        if bias is not None:
            ref = O.round_to(ref + bias, tag)
        assert np.array_equal(torch_to_bits(y), O.from_f32(ref, tag)), name
        return
    assert K % 64 in (16, 32, 48)
    s = O.round_to(rng.random(N, dtype=np.float32) / 1e2 + 1e-4, tag)
    s_t = bits_to_torch(O.from_f32(s, tag), tag)
    if fam == "fp8":
        ak, wk = var
        a_bits = _fp8_codes(ak, (M, K), rng, 1.0)
        w_bits = _fp8_codes(wk, (N, K), rng, 2.0)
        with _overrides(ovr):
            y, family = cabi_qbytes_mm(bits_to_torch(a_bits, ak), bits_to_torch(w_bits, wk), s_t)
            torch.cuda.synchronize()
        assert family == 1, name
        _check_fp8_native(y, a_bits, ak, w_bits, wk, s, tag, name)
        return
    wk = var
    a = O.round_to(rng.standard_normal((M, K), dtype=np.float32), tag)
    if wk == "int8":
        w_store = rng.integers(-128, 128, size=(N, K), dtype=np.int8)
        w = w_store.astype(np.float32)
    else:
        w_store = _fnuz_all_codes(N, K, rng) if wk == "e4m3fnuz" else _fp8_codes(wk, (N, K), rng)
        w = O.fp8_bits_to_f32(w_store, wk)
    with _overrides(ovr):
        y, family = cabi_qbytes_mm(bits_to_torch(O.from_f32(a, tag), tag), bits_to_torch(w_store, wk), s_t, bias_t)
        torch.cuda.synchronize()
    assert family == 1, name
    _check_weight_only(y, a, w, s, bias, tag, name)


# --------------------------------------------------------------------------------- many tiles per CTA, short K
# M = 2048 and N ~ 4096 give hundreds of output tiles over the SMs, while K spans one or two k-blocks: fewer than the three
# pipeline stages, so each staging group starts tiles ahead of the consumers (f_tile = blockIdx.x + (grp / kblocks) *
# gridDim.x) and its stepping loop skips several tiles at a time.
SHORT_K = [("int4", 32), ("int4", 64), ("int4", 128), ("int8", 16), ("int8", 48), ("int8", 64), ("int8", 208),
           ("fp8", 16), ("fp8", 48), ("fp8", 64), ("fp8", 112), ("w8", 16), ("w8", 48), ("w8", 64), ("w8", 112)]


@pytest.mark.parametrize("fam,K", SHORT_K, ids=[f"{f}-k{k}" for f, k in SHORT_K])
def test_many_tiles_short_k(fam, K):
    M, tag = 2048, "bf16"
    rng = np.random.default_rng(K + len(fam))
    rows = band_rows(M, seed=K)
    lib = native().load()
    if fam == "int4":
        N, G = 4000, K  # N / 2 % 64 == 16
        _, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=K)
        x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
        deq_bits = O.dequantize_qbits(packed, 4, scale, shift, tag, N, K, G)
        dev_x, dev_p = bits_to_torch(x_bits, tag), torch.from_numpy(packed).cuda()
        dev_s, dev_z = bits_to_torch(scale, tag), bits_to_torch(shift, tag)
        y = cabi_qbits_mm(dev_x, dev_p, dev_s, dev_z, None, N, K, G)
        assert lib.qb200_last_kernel_family() == 1
        deq_gpu = cabi_dequantize_qbits(dev_p, dev_s, dev_z, N, K, G, 4)
        torch.cuda.synchronize()
        assert np.array_equal(torch_to_bits(deq_gpu), deq_bits)
        check_linear(y[torch.from_numpy(rows).cuda()], x_bits[rows], deq_bits, None, tag, (fam, K))
        check_full_against_device_fp32(y, dev_x, deq_gpu, None, (fam, K))
        return
    N = 4095
    if fam == "int8":
        A = rng.integers(-128, 128, size=(M, K), dtype=np.int8)
        W = rng.integers(-128, 128, size=(N, K), dtype=np.int8)
        s = O.round_to(rng.random(N, dtype=np.float32) / 1e3 + 1e-5, tag)
        At, Wt, st = torch.from_numpy(A).cuda(), torch.from_numpy(W).cuda(), bits_to_torch(O.from_f32(s, tag), tag)
        y, family = cabi_qbytes_mm(At, Wt, st)
        torch.cuda.synchronize()
        assert family == 1
        ref = O.qbytes_int_mm(A[rows], W, s, tag)
        assert np.array_equal(torch_to_bits(y[torch.from_numpy(rows).cuda()]), ref)
        acc = torch.matmul(At.double(), Wt.double().t())  # exact: |acc| < 2^24
        full = (acc.float() * st.float().reshape(1, -1)).to(torch.bfloat16)
        assert torch.equal(y, full), int((y != full).sum())
        return
    s = O.round_to(rng.random(N, dtype=np.float32) / 1e2 + 1e-4, tag)
    st = bits_to_torch(O.from_f32(s, tag), tag)
    if fam == "fp8":
        a_bits = _fp8_codes("e4m3fn", (M, K), rng, 1.0)
        w_bits = _fp8_codes("e4m3fn", (N, K), rng, 2.0)
        At, Wt = bits_to_torch(a_bits, "e4m3fn"), bits_to_torch(w_bits, "e4m3fn")
        y, family = cabi_qbytes_mm(At, Wt, st)
        torch.cuda.synchronize()
        assert family == 1
        _check_fp8_native(y[torch.from_numpy(rows).cuda()], a_bits[rows], "e4m3fn", w_bits, "e4m3fn", s, tag, (fam, K))
        check_full_against_device_fp32(y, At.float(), Wt.float() * st.float().reshape(-1, 1), None, (fam, K))
        return
    a = O.round_to(rng.standard_normal((M, K), dtype=np.float32), tag)
    w_bits = _fp8_codes("e5m2", (N, K), rng)
    At, Wt = bits_to_torch(O.from_f32(a, tag), tag), bits_to_torch(w_bits, "e5m2")
    y, family = cabi_qbytes_mm(At, Wt, st)
    torch.cuda.synchronize()
    assert family == 1
    _check_weight_only(y[torch.from_numpy(rows).cuda()], a[rows], O.fp8_bits_to_f32(w_bits, "e5m2"), s, None, tag, (fam, K))
    ws_t = (st.reshape(-1, 1) * Wt.to(torch.bfloat16)).to(torch.bfloat16)  # the reference's operand, on the device
    check_full_against_device_fp32(y, At, ws_t, None, (fam, K))


# --------------------------------------------------------------------------------- int4 groups 192 / 320
@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("G,zp", [(192, False), (320, False), (192, True)])
@pytest.mark.parametrize("K", [960, 1920])
def test_int4_non_power_of_two_groups(tag, G, zp, K):
    """Groups that are multiples of 64 but not powers of two take the division path (group_log2 = -1) in the staging warps
    and the gemvs: decode sizes through the automatic route (with and without a workspace), M = 12 (the wgmma kernel behind
    the gemvs) and both tile heights."""
    N = 640
    _, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=G + K, zeropoint=zp)
    deq_bits = O.dequantize_qbits(packed, 4, scale, shift, tag, N, K, G, shift_is_int=zp)
    dev_p, dev_s = torch.from_numpy(packed).cuda(), bits_to_torch(scale, tag)
    dev_z = torch.from_numpy(shift).cuda() if zp else bits_to_torch(shift, tag)
    assert np.array_equal(torch_to_bits(cabi_dequantize_qbits(dev_p, dev_s, dev_z, N, K, G, 4)), deq_bits)
    lib = native().load()
    rng = np.random.default_rng(G * 7 + K)
    runs = [(M, ws, None) for M in (1, 5, 8) for ws in (True, False)] + [(12, True, None)]
    runs += [(M, True, tm) for M in (33, 300) for tm in (64, 128)]
    for M, ws, tm in runs:
        x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
        bias_bits = O.from_f32(rng.standard_normal(N, dtype=np.float32), tag) if M % 2 else None
        with _overrides([("OVR_TILE_M", tm)] if tm else []):
            y = cabi_qbits_mm(bits_to_torch(x_bits, tag), dev_p, dev_s, dev_z,
                              None if bias_bits is None else bits_to_torch(bias_bits, tag), N, K, G, use_workspace=ws)
            family = lib.qb200_last_kernel_family()
            torch.cuda.synchronize()
        if tm:
            assert family == 1, (M, tm)
        check_linear(y, x_bits, deq_bits, bias_bits, tag, (G, zp, K, M, ws, tm, family))


# --------------------------------------------------------------------------------- NaN weight codes
@pytest.mark.parametrize("wkind,nan_code", [("e4m3fnuz", 0x80), ("e4m3fn", 0x7F), ("e5m2", 0x7E)])
@pytest.mark.parametrize("route", ["tensor", "cuda-core"])
def test_nan_weight_code_gives_one_nan_column(wkind, nan_code, route):
    M, N, K, tag = 70, 200, 256, "bf16"
    rng = np.random.default_rng(31)
    a = O.round_to(rng.standard_normal((M, K), dtype=np.float32), tag)
    w_bits = _fnuz_all_codes(N, K, rng) if wkind == "e4m3fnuz" else _fp8_codes(wkind, (N, K), rng)
    n_nan, k_nan = 77, 131
    w_bits[n_nan, k_nan] = nan_code
    s = O.round_to(rng.random(N, dtype=np.float32) / 1e2 + 1e-4, tag)
    ovr = [("OVR_QBYTES_ROUTE", native().ROUTE_QBYTES_SIMT)] if route == "cuda-core" else []
    with _overrides(ovr):
        y, family = cabi_qbytes_mm(bits_to_torch(O.from_f32(a, tag), tag), bits_to_torch(w_bits, wkind),
                                   bits_to_torch(O.from_f32(s, tag), tag))
        torch.cuda.synchronize()
    assert family == (1 if route == "tensor" else 2)
    yf = torch_to_f32(y)
    assert np.isnan(yf[:, n_nan]).all()
    others = np.delete(np.arange(N), n_nan)
    assert np.isfinite(yf[:, others]).all()
    w = O.fp8_bits_to_f32(w_bits, wkind)
    _check_weight_only(y[:, torch.from_numpy(others).cuda()], a, w[others], s[others], None, tag, (wkind, route))
