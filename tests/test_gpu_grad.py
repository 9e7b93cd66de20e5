"""Input gradient of the quantized linears on the wgmma kernel (gemm_tc_dgrad.cuh): dX = gO @ dequant(W).

The parity contract: the operands are bit-identical to the reference's (gO as given, dequantize() exactly) and only the
fp32 summation order is free, so |dX - dX64| <= 0.5 ulp + 2^-22 sqrt(N) (|gO| @ |Wd|)  (helpers.check_linear with gO as
the activations and Wd^T as the weight).

* Census: every instantiation (int4: dtype x shift kind x tile rows; 8-bit: dtype x weight format x tile rows), forced by
  the tile override, one row past a tile boundary, with a reduction tail ((N/2) % 64 != 0 or N % 128 != 0) and a K tail.
* Llama shapes at M = 4096 against the fp64 oracle on a band of rows and against the composition on every element.
* int4 group sizes 32 .. 320 at small and ragged M.
* The nibble-plane boundary: +-Inf entries of gO at columns N/2 - 1 and N/2 give the composition's Inf / NaN pattern.
* Autograd through QLinear (frozen and unfrozen), the reference's stored gradients (tests/golden/grad.npz) and the shapes
  the kernel declines (2-bit, fp32), which keep the composition.
"""
import contextlib
import os

import numpy as np
import pytest
import torch

import quanto_b200 as q
from helpers import (O, band_rows, bits_to_torch, cabi_dequantize_qbits, check_full_against_device_fp32, check_linear,
                     native, torch_to_bits, torch_to_f32)
from quanto_b200.tensor import function as qfunction

pytestmark = pytest.mark.gpu
TDT = {"f16": torch.float16, "bf16": torch.bfloat16, "f32": torch.float32}
F8 = {"e4m3fn": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2, "e4m3fnuz": torch.float8_e4m3fnuz}


@contextlib.contextmanager
def _tile(rows):
    n = native()
    with n.test_override(n.OVR_TILE_M, rows):
        yield


def _int4_weights(N, K, G, dtype, zp, seed):
    """Random canonical int4 storage on the device: any byte is a valid pair of nibbles."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    rows = N * K // G
    packed = torch.randint(0, 256, (rows // 2, G), dtype=torch.uint8, device="cuda", generator=gen)
    scale = (torch.rand(rows, 1, device="cuda", generator=gen) * 0.01 + 0.002).to(dtype)
    if zp:
        shift = torch.randint(0, 16, (rows, 1), dtype=torch.uint8, device="cuda", generator=gen)
    else:
        shift = (scale.float() * (7.0 + 2 * torch.rand(rows, 1, device="cuda", generator=gen))).to(dtype)
    return packed, scale, shift


def _grad_out(M, N, dtype, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(M, N, device="cuda", generator=gen).to(dtype)


def cabi_qbits_grad(gO, packed, scale, shift, N, K, G):
    n = native()
    lib = n.load()
    out = torch.empty((gO.shape[0], K), dtype=gO.dtype, device=gO.device)
    sh = shift.reshape(-1).contiguous()
    n.check(lib.qb200_qbits_mm_grad_input(n.ptr(gO), n.ptr(packed), n.ptr(scale), n.ptr(sh), n.ptr(out), gO.shape[0], N,
                                          K, G, n.DTYPE_CODE[gO.dtype], 0 if sh.dtype.is_floating_point else 1,
                                          n.stream_ptr(gO.device)), "qbits_mm_grad_input")
    return out, lib.qb200_last_kernel_family()


def cabi_qbytes_grad(gO, w, scales):
    n = native()
    lib = n.load()
    N, K = w.shape
    out = torch.empty((gO.shape[0], K), dtype=gO.dtype, device=gO.device)
    n.check(lib.qb200_qbytes_mm_grad_input(n.ptr(gO), n.ptr(w), n.ptr(scales.reshape(-1).contiguous()), n.ptr(out),
                                           gO.shape[0], N, K, n.DTYPE_CODE[w.dtype], n.DTYPE_CODE[gO.dtype],
                                           n.stream_ptr(gO.device)), "qbytes_mm_grad_input")
    return out, lib.qb200_last_kernel_family()


def _check_int4(M, N, K, G, tag, zp, seed, label):
    dtype = TDT[tag]
    packed, scale, shift = _int4_weights(N, K, G, dtype, zp, seed)
    gO = _grad_out(M, N, dtype, seed + 1)
    dx, fam = cabi_qbits_grad(gO, packed, scale, shift, N, K, G)
    torch.cuda.synchronize()
    assert fam == 1, label
    wd = cabi_dequantize_qbits(packed, scale, shift, N, K, G, 4)  # bit-exact with the oracle (test_gpu_cabi)
    check_linear(dx, torch_to_bits(gO), torch_to_bits(wd).T, None, tag, label)
    return dx, gO, wd


def _bytes_weights(N, K, wkind, tag, seed):
    gen = torch.Generator().manual_seed(seed)
    if wkind == "int8":
        w = torch.randint(-127, 128, (N, K), dtype=torch.int8, generator=gen)
        wf = w.numpy().astype(np.float32)
    else:
        lim = 240.0 if wkind == "e4m3fnuz" else 448.0
        w = (torch.randn(N, K, generator=gen) * 30).clamp(-lim, lim).to(F8[wkind])
        wf = O.fp8_bits_to_f32(w.view(torch.uint8).numpy(), wkind)
    s_bits = O.from_f32(torch.rand(N, generator=gen).numpy().astype(np.float32) * 0.01 + 0.001, tag)
    wd = O.round_to(O.to_f32(s_bits, tag).reshape(-1, 1) * wf, tag)  # QBytesDequantizer: rnd(scale * W)
    return w.cuda(), bits_to_torch(s_bits, tag), wd


# --------------------------------------------------------------------------------------------------------- census
@pytest.mark.parametrize("rows", [64, 128])
@pytest.mark.parametrize("zp", [False, True], ids=["float-shift", "zero-point"])
@pytest.mark.parametrize("tag", ["bf16", "f16"])
def test_census_int4(tag, zp, rows):
    # (N/2) % 64 = 8: a zero-filled reduction tail in both planes; K % 128 = 64: a tile whose second half is past K
    G = 64 if tag == "bf16" else 32
    with _tile(rows):
        _check_int4(rows + 1, 272, 448, G, tag, zp, 11, ("int4", tag, zp, rows))


@pytest.mark.parametrize("rows", [64, 128])
@pytest.mark.parametrize("wkind", ["int8", "e4m3fn", "e5m2", "e4m3fnuz"])
@pytest.mark.parametrize("tag", ["bf16", "f16"])
def test_census_8bit(tag, wkind, rows):
    M, N, K = rows + 1, 136, 448  # N % 128 = 8, K % 128 = 64
    w, s, wd = _bytes_weights(N, K, wkind, tag, 5)
    gO = _grad_out(M, N, TDT[tag], 6)
    with _tile(rows):
        dx, fam = cabi_qbytes_grad(gO, w, s)
    torch.cuda.synchronize()
    assert fam == 1
    check_linear(dx, torch_to_bits(gO), O.from_f32(wd.T, tag), None, tag, (wkind, tag, rows))


# ---------------------------------------------------------------------------------------------------- Llama shapes
@pytest.mark.parametrize("zp", [False, True], ids=["float-shift", "zero-point"])
@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("N,K", [(14336, 4096), (4096, 14336)])
def test_llama_shapes(N, K, tag, zp):
    M, G = 4096, 128
    dtype = TDT[tag]
    packed, scale, shift = _int4_weights(N, K, G, dtype, zp, 21)
    gO = _grad_out(M, N, dtype, 22)
    dx, fam = cabi_qbits_grad(gO, packed, scale, shift, N, K, G)
    assert fam == 1
    wd = cabi_dequantize_qbits(packed, scale, shift, N, K, G, 4)
    # every element against the fp32 product of the same operands (a misplaced or stale tile anywhere)
    check_full_against_device_fp32(dx, gO, wd.t(), None, ("llama", N, K, tag, zp))
    comp = torch.matmul(gO, wd)  # the composition the backward ran before: dequantize, then a dense GEMM
    assert float((dx.float() - comp.float()).norm() / comp.float().norm()) < 1e-3
    # the fp64 oracle on a band of rows (every tile row band sampled) -- for one shift kind per dtype
    if zp == (tag == "f16"):
        rows = band_rows(M, seed=N + K, per_band=1)
        ridx = torch.from_numpy(rows).cuda()
        check_linear(dx[ridx], torch_to_bits(gO[ridx]), torch_to_bits(wd.t().contiguous()), None, tag,
                     ("llama band", N, K, tag, zp))


# ------------------------------------------------------------------------------------------- groups and small M
@pytest.mark.parametrize("G", [32, 64, 128, 192, 320])
def test_int4_groups_small_m(G):
    K = 896 if G == 128 else 960
    for M in (1, 5, 64, 65, 300):
        _check_int4(M, 144, K, G, "bf16" if M % 2 else "f16", M == 65, 100 + G + M, ("group", G, M))


# ------------------------------------------------------------------------------------------------ plane boundary
@pytest.mark.parametrize("rows", [64, 128])
def test_plane_boundary_inf(rows):
    """+-Inf at gO columns N/2 - 1 and N/2: a box of one plane that read into the other plane, or a reduction tail that
    was not zero-filled, turns the Inf into NaN where the composition has none (and vice versa)."""
    M, N, K, G = 70, 272, 256, 128
    packed, scale, shift = _int4_weights(N, K, G, torch.bfloat16, False, 31)
    gO = _grad_out(M, N, torch.bfloat16, 32)
    gO[3, N // 2 - 1] = float("inf")
    gO[3, N // 2] = float("-inf")
    gO[40, N // 2] = float("inf")
    gO[66, N // 2 - 1] = float("-inf")
    with _tile(rows):
        dx, _ = cabi_qbits_grad(gO, packed, scale, shift, N, K, G)
    ref = torch.matmul(gO, cabi_dequantize_qbits(packed, scale, shift, N, K, G, 4))
    torch.cuda.synchronize()
    assert torch.equal(torch.isnan(dx), torch.isnan(ref))
    assert torch.equal(torch.isposinf(dx), torch.isposinf(ref))
    assert torch.equal(torch.isneginf(dx), torch.isneginf(ref))
    assert int(torch.isnan(dx).sum()) > 0 and int(torch.isinf(dx).sum()) > 0
    finite = torch.isfinite(ref)
    assert bool(torch.isfinite(dx[finite]).all())
    finite_rows = torch.isfinite(ref).all(dim=1)
    check_linear(dx[finite_rows], torch_to_bits(gO[finite_rows]),
                 torch_to_bits(cabi_dequantize_qbits(packed, scale, shift, N, K, G, 4).t().contiguous()), None, "bf16",
                 "plane boundary, finite rows")


# ------------------------------------------------------------------------------------------------------- autograd
@contextlib.contextmanager
def _record_families():
    """Record qb200_last_kernel_family() right after every input-gradient op, on the thread that ran it (the autograd
    engine runs CUDA backward on its own thread; the family is thread-local)."""
    lib = native().load()
    seen = []
    orig = (qfunction.qbits_grad_input, qfunction.qbytes_grad_input)

    def wrap(fn):
        def inner(gO, other):
            out = fn(gO, other)
            seen.append(lib.qb200_last_kernel_family() if out is not None else None)
            return out
        return inner

    qfunction.qbits_grad_input, qfunction.qbytes_grad_input = wrap(orig[0]), wrap(orig[1])
    try:
        yield seen
    finally:
        qfunction.qbits_grad_input, qfunction.qbytes_grad_input = orig


def _frozen_qlinear(wq, K, N, dtype, seed, bias=True):
    torch.manual_seed(seed)
    lin = torch.nn.Linear(K, N, bias=bias).to(dtype).cuda()
    with torch.no_grad():
        lin.weight.mul_(2.0)
    ql = q.QLinear.from_module(lin, weights=wq)
    ql.freeze()
    return ql


def _dequantized(ql):
    with torch.no_grad():
        return ql.weight.dequantize()


@pytest.mark.parametrize("wq", ["qint4", "qint8", "qfloat8"])
def test_autograd_frozen_qlinear(wq):
    tag = "bf16"
    M, K, N = 37, 512, 384
    ql = _frozen_qlinear(q.qtypes[wq], K, N, torch.bfloat16, 41)
    x = torch.randn(3, M, K, device="cuda").to(torch.bfloat16).requires_grad_(True)  # 3 * 37 rows: the native route
    y = ql(x)
    gO = torch.randn_like(y)
    with _record_families() as fams:
        y.backward(gO)
    torch.cuda.synchronize()
    assert fams == [1], fams
    wd = _dequantized(ql)
    check_linear(x.grad.reshape(-1, K), torch_to_bits(gO.reshape(-1, N)), torch_to_bits(wd.t().contiguous()), None, tag,
                 ("autograd", wq))
    assert torch.equal(ql.bias.grad, gO.sum((0, 1)))


@pytest.mark.parametrize("wq", ["qint4", "qint8"])
def test_autograd_unfrozen_weight_and_bias_grads_keep_their_formulas(wq):
    M, K, N = 64, 256, 192
    torch.manual_seed(43)
    lin = torch.nn.Linear(K, N).to(torch.bfloat16).cuda()
    ql = q.QLinear.from_module(lin, weights=q.qtypes[wq])
    x = torch.randn(M, K, device="cuda").to(torch.bfloat16).requires_grad_(True)
    y = ql(x)
    gO = torch.randn_like(y)
    with _record_families() as fams:
        y.backward(gO)
    assert fams == [1], fams
    assert torch.equal(ql.weight.grad, torch.matmul(gO.t(), x.detach()))
    assert torch.equal(ql.bias.grad, gO.sum(0))
    assert ql.weight.grad.dtype == torch.bfloat16 and x.grad.shape == x.shape


@pytest.mark.parametrize("wq", ["qint4", "qint8"])
def test_above_the_crossover_the_backward_composes(wq):
    """Above NATIVE_GRAD_INPUT_MAX_M rows the composition is faster (DESIGN section 6): the base formula runs."""
    M = qfunction.NATIVE_GRAD_INPUT_MAX_M + 1
    ql = _frozen_qlinear(q.qtypes[wq], 256, 128, torch.bfloat16, 47)
    x = torch.randn(M, 256, device="cuda").to(torch.bfloat16).requires_grad_(True)
    y = ql(x)
    gO = torch.randn_like(y)
    with _record_families() as fams:
        y.backward(gO)
    assert fams == [None], fams
    assert torch.equal(x.grad, torch.matmul(gO, _dequantized(ql)))


def test_declined_shapes_keep_the_composition():
    # 2-bit weights and fp32 gradients: the kernel declines, the op composes dequantize + matmul
    for wq, dtype, tag in ((q.qint2, torch.bfloat16, "bf16"), (q.qint4, torch.float32, "f32")):
        ql = _frozen_qlinear(wq, 256, 128, dtype, 51)
        x = torch.randn(33, 256, device="cuda").to(dtype).requires_grad_(True)
        y = ql(x)
        gO = torch.randn_like(y)
        with _record_families() as fams:
            y.backward(gO)
        if dtype == torch.float32:
            assert fams == [0], fams  # the C ABI was called and declined
        ref = torch.matmul(gO, _dequantized(ql))
        assert torch.equal(x.grad, ref), (wq, dtype)


def test_fixture_replay(golden_dir):
    """The reference's own autograd (CPU) against this library's (CUDA) on the stored layers and gO."""
    z = np.load(os.path.join(golden_dir, "grad.npz"))

    def rel(a, ref_bits, tag):
        ref = O.to_f32(ref_bits, tag).astype(np.float64)
        return np.linalg.norm(torch_to_f32(a).astype(np.float64) - ref) / np.linalg.norm(ref)

    for i in range(int(z["n"])):
        p = f"g{i}_"
        tag = str(z[p + "tag"])
        dtype = TDT[tag]
        N, K, M, G = (int(v) for v in z[p + "shape"])
        wq = q.qtypes[str(z[p + "wq"])]
        lin = torch.nn.Linear(K, N, bias=True).to(dtype)
        frozen = bool(int(z[p + "frozen"]))
        if not frozen:
            with torch.no_grad():
                lin.weight.copy_(bits_to_torch(z[p + "weight"], tag, device="cpu"))
        with torch.no_grad():
            lin.bias.copy_(bits_to_torch(z[p + "bias"], tag, device="cpu"))
        ql = q.QLinear.from_module(lin, weights=wq)
        if frozen:
            sd = {"bias": bits_to_torch(z[p + "bias"], tag, device="cpu")}
            for key in z.files:
                if key.startswith(p + "sd_"):
                    name, arr = key[len(p) + 3:], z[key]
                    if name.endswith("_data") and wq.bits == 8 and wq.is_floating_point:
                        sd[name] = torch.from_numpy(arr.copy()).view(wq.dtype)
                    elif name.endswith("_data") or arr.dtype == np.uint8:
                        sd[name] = torch.from_numpy(arr.copy())
                    else:
                        sd[name] = bits_to_torch(arr, tag, device="cpu")
            ql.load_state_dict(sd)
            ql.weight.requires_grad_(False)
        ql = ql.cuda()
        x = bits_to_torch(z[p + "x"], tag).requires_grad_(True)
        y = ql(x)
        y.backward(bits_to_torch(z[p + "gO"], tag))
        torch.cuda.synchronize()
        assert rel(x.grad, z[p + "x_grad"], tag) < 1e-3, (i, "x.grad", rel(x.grad, z[p + "x_grad"], tag))
        assert rel(ql.bias.grad, z[p + "bias_grad"], tag) < 1e-3, (i, "bias.grad")
        if not frozen:
            assert rel(ql.weight.grad, z[p + "weight_grad"], tag) < 1e-3, (i, "weight.grad")
