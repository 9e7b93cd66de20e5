"""Parity at the configurations bench.py measures (BASELINE.json configs[1..3]) and on every shipped instantiation.

The small-shape suites (test_gpu_cabi.py) never make a persistent CTA process more than one tile; these tests run the
Llama-3-8B shapes (M = 4096, N = 14336 / 4096, K = 4096 / 14336), where every CTA loops over 2-7 tiles: accumulator
mbarrier phase wrap, the staging groups' tile stepping and both tile heights (one or two consumer warpgroups) are all
executed and checked.

How a 4096 x 14336 x 4096 product is checked against the CPU oracle in seconds:
* the operands: the kernel's dequantisation is bit-exact against the oracle on the WHOLE weight (the standalone
  dequantize entry point shares the device arithmetic of the GEMM's staging warps);
* the GEMM: float64 oracle on a row sample that contains two rows of every 32-row band of M -- every output tile, every
  epilogue warp and every column chunk of every tile is checked -- with the per-element bound of test_gpu_cabi.py;
* the full output, all 58.7 M elements: against an fp32 product of the same (verified) operands computed on the device,
  rounded like the reference rounds (a cross-check for misplaced tiles; the oracle sample above is the parity check);
* int8 x int8: bit-exact on the row sample against the oracle, and bit-exact on the full output against the same
  integer product evaluated in float64 on the device.
Reference assertions these strengthen: tests/library/test_mm.py:35-49, tests/tensor/weights/weight_helpers.py:19-37.
"""
import numpy as np
import pytest
import torch

from helpers import (O, band_rows, bits_to_torch, cabi_dequantize_qbits, cabi_qbits_mm, cabi_qbytes_mm,
                     check_full_against_device_fp32, make_qbits_weights, native, torch_to_bits, torch_to_f32)

pytestmark = pytest.mark.gpu


class RowOracle:
    """The test_gpu_cabi._check_linear bound on a row sample (float64 oracle, all columns), computed once per case."""

    def __init__(self, rows, x_bits, deq_bits, bias_bits, tag):
        x = O.to_f32(x_bits[rows], tag)
        w = O.to_f32(deq_bits, tag)
        bias = None if bias_bits is None else O.to_f32(bias_bits, tag)
        self.rows = rows
        self.y64, y_ref, tol = O.linear_from_dequantized(x, w, bias, tag)
        self.bound = 1.02 * tol + O.accumulate_allowance(x, w)
        self.yr = O.to_f32(y_ref, tag).astype(np.float64)

    def check(self, y_gpu, label):
        y = torch_to_f32(y_gpu[torch.from_numpy(self.rows).to(y_gpu.device)]).astype(np.float64)
        err = np.abs(y - self.y64)
        assert np.all(err <= self.bound), (label, float(np.max(err / self.bound)),
                                           np.unravel_index(np.argmax(err / self.bound), err.shape))
        rel = np.linalg.norm(y - self.yr) / max(np.linalg.norm(self.yr), 1e-30)
        assert rel < 1e-3, (label, rel)


def check_rows_linear(y_gpu, rows, x_bits, deq_bits, bias_bits, tag, label):
    RowOracle(rows, x_bits, deq_bits, bias_bits, tag).check(y_gpu, label)


def int4_case(M, N, K, G, tag, zeropoint, bias, seed):
    q, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=seed, zeropoint=zeropoint)
    rng = np.random.default_rng(seed + 17)
    x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
    bias_bits = O.from_f32(rng.standard_normal(N, dtype=np.float32), tag) if bias else None
    deq_bits = O.dequantize_qbits(packed, 4, scale, shift, tag, N, K, G, shift_is_int=zeropoint)
    shift_t = torch.from_numpy(shift).cuda() if zeropoint else bits_to_torch(shift, tag)
    dev = dict(x=bits_to_torch(x_bits, tag), packed=torch.from_numpy(packed).cuda(), scale=bits_to_torch(scale, tag),
               shift=shift_t, bias=None if bias_bits is None else bits_to_torch(bias_bits, tag))
    # operands: bit-exact on the whole weight
    deq_gpu = cabi_dequantize_qbits(dev["packed"], dev["scale"], dev["shift"], N, K, G, 4)
    assert np.array_equal(torch_to_bits(deq_gpu), deq_bits), "dequantised operand differs from the oracle"
    return x_bits, deq_bits, bias_bits, dev, deq_gpu


INT4_CASES = [
    # (M, N, K, tag, zeropoint, bias)
    (4096, 14336, 4096, "bf16", False, False),   # BASELINE configs[1], the bench default
    (4096, 4096, 14336, "bf16", False, True),    # down projection
    (4096, 14336, 4096, "f16", True, True),
    (4096, 4096, 14336, "f16", False, False),
]
# kernel variants: (label, override key, value) -- every one must give the same operands and pass the same bounds
INT4_VARIANTS = [
    ("auto", None, None),
    ("tile_m64", "OVR_TILE_M", 64),
    ("tile_m128", "OVR_TILE_M", 128),
]


@pytest.mark.parametrize("M,N,K,tag,zeropoint,bias", INT4_CASES)
def test_int4_bench_shapes_all_kernel_variants(M, N, K, tag, zeropoint, bias):
    n = native()
    lib = n.load()
    x_bits, deq_bits, bias_bits, dev, deq_gpu = int4_case(M, N, K, 128, tag, zeropoint, bias, seed=M + N + K)
    oracle = RowOracle(band_rows(M, seed=N), x_bits, deq_bits, bias_bits, tag)
    outs = {}
    for label, key, value in INT4_VARIANTS:
        keys = key if isinstance(key, tuple) else ((key,) if key else ())
        vals = value if isinstance(value, tuple) else ((value,) if key else ())
        try:
            for k_, v_ in zip(keys, vals):
                n.check(lib.qb200_test_override(getattr(n, k_), v_), "override")
            y = cabi_qbits_mm(dev["x"], dev["packed"], dev["scale"], dev["shift"], dev["bias"], N, K, 128)
            torch.cuda.synchronize()
            assert lib.qb200_last_kernel_family() == 1
        finally:
            for k_ in keys:
                lib.qb200_test_override(getattr(n, k_), 0)
        oracle.check(y, (label, M, N, K, tag))
        check_full_against_device_fp32(y, dev["x"], deq_gpu, dev["bias"], (label, M, N, K, tag))
        outs[label] = y
    # same operands, same k order inside a tile: both tile heights are bit-identical to each other
    assert torch.equal(outs["tile_m64"], outs["tile_m128"])
    # through the QTensor / F.linear surface: the same launch
    import quanto_b200 as q
    rows_g = N * K // 128
    w = q.WeightQBitsTensor(q.qint4, 0, 128, torch.Size([N, K]), (K, 1),
                            q.PackedTensor(dev["packed"], 4, torch.Size([rows_g, 128]), (128, 1)),
                            dev["scale"].reshape(-1, 1), dev["shift"].reshape(-1, 1))
    y_lin = torch.nn.functional.linear(dev["x"], w, dev["bias"])
    assert torch.equal(y_lin, outs["auto"])


@pytest.mark.parametrize("M", [33, 64, 100, 128])
@pytest.mark.parametrize("tag", ["bf16", "f16"])
def test_int4_mid_m_llama_shapes(M, tag):
    """32 < M <= 128: the wgmma kernel (one or two consumer warpgroups), at N = 14336 and K = 14336."""
    n = native()
    lib = n.load()
    for (N, K) in ((14336, 4096), (4096, 14336)):
        if tag == "f16" and K == 14336:
            continue
        x_bits, deq_bits, bias_bits, dev, deq_gpu = int4_case(M, N, K, 128, tag, M == 100, M % 2 == 1, seed=M + N)
        y = cabi_qbits_mm(dev["x"], dev["packed"], dev["scale"], dev["shift"], dev["bias"], N, K, 128)
        y2 = cabi_qbits_mm(dev["x"], dev["packed"], dev["scale"], dev["shift"], dev["bias"], N, K, 128)
        torch.cuda.synchronize()
        assert lib.qb200_last_kernel_family() == 1 and torch.equal(y, y2)
        rows = np.arange(M)
        check_rows_linear(y, rows, x_bits, deq_bits, bias_bits, tag, ("tcdecode", M, N, K, tag))


@pytest.mark.parametrize("M", [9, 16, 32])
def test_int4_small_m_routes_agree(M):
    """8 < M <= 32 at N = 14336: whichever kernel the dispatcher picks, and the other candidates, pass the same bound."""
    n = native()
    lib = n.load()
    N, K, tag = 14336, 4096, "bf16"
    x_bits, deq_bits, bias_bits, dev, _ = int4_case(M, N, K, 128, tag, False, M == 16, seed=M)
    oracle = RowOracle(np.arange(M), x_bits, deq_bits, bias_bits, tag)
    routes = (0, n.ROUTE_INT4_GEMV, n.ROUTE_INT4_GENERAL) + ((n.ROUTE_INT4_RING2,) if M <= 16 else ())
    for route in routes:
        with n.test_override(n.OVR_INT4_ROUTE, route):
            y = cabi_qbits_mm(dev["x"], dev["packed"], dev["scale"], dev["shift"], dev["bias"], N, K, 128)
            torch.cuda.synchronize()
        oracle.check(y, ("route", route, M))


@pytest.mark.parametrize("pmode", [1, 2, 3])
@pytest.mark.parametrize("M", [1, 8])
def test_int4_ring_gemv_producer_modes(M, pmode):
    """The TMA-ring gemv gives the same bits whichever lanes issue the copies.  The automatic route runs this shape on the
    second-generation ring kernel, which has no producer modes: the first generation is forced for every run."""
    n = native()
    N, K, tag = 14336, 4096, "bf16"
    x_bits, deq_bits, bias_bits, dev, _ = int4_case(M, N, K, 128, tag, False, False, seed=M)
    with n.test_override(n.OVR_INT4_ROUTE, n.ROUTE_INT4_RING):
        y0 = cabi_qbits_mm(dev["x"], dev["packed"], dev["scale"], dev["shift"], dev["bias"], N, K, 128)
        with n.test_override(n.OVR_GEMV_PRODUCER, pmode):
            y1 = cabi_qbits_mm(dev["x"], dev["packed"], dev["scale"], dev["shift"], dev["bias"], N, K, 128)
            torch.cuda.synchronize()
    assert n.load().qb200_last_kernel_family() == 3
    assert torch.equal(y0, y1)
    check_rows_linear(y1, np.arange(M), x_bits, deq_bits, bias_bits, tag, ("ring", pmode, M))


# ------------------------------------------------------------------------------------------ int8 / fp8 / weight-only
def _int_product_on_device(A, W):
    """Exact integer product evaluated in float64 on the device (|sum| < 2^53): the full-output cross-check."""
    return torch.matmul(A.double(), W.double().t())


@pytest.mark.parametrize("N", [4096, 14336])
@pytest.mark.parametrize("variant", ["auto", "tile128", "tile256", "tile_m64"])
def test_int8_bench_shapes_bit_exact(N, variant):
    n = native()
    lib = n.load()
    M, K, tag = 4096, 4096, "bf16"
    rng = np.random.default_rng(N)
    A = rng.integers(-127, 128, size=(M, K), dtype=np.int8)
    W = rng.integers(-128, 128, size=(N, K), dtype=np.int8)
    s = O.round_to(rng.random(N, dtype=np.float32) / 1e3 + 1e-5, tag)
    bias = O.round_to(rng.standard_normal(N, dtype=np.float32), tag) if N == 14336 else None
    At, Wt = torch.from_numpy(A).cuda(), torch.from_numpy(W).cuda()
    st = bits_to_torch(O.from_f32(s, tag), tag)
    bt = None if bias is None else bits_to_torch(O.from_f32(bias, tag), tag)
    key, val = {"auto": (None, 0), "tile128": (n.OVR_QBYTES_TILE_N, 128), "tile256": (n.OVR_QBYTES_TILE_N, 256),
                "tile_m64": (n.OVR_TILE_M, 64)}[variant]
    try:
        if key is not None:
            lib.qb200_test_override(key, val)
        y, family = cabi_qbytes_mm(At, Wt, st, bt)
        torch.cuda.synchronize()
    finally:
        if key is not None:
            lib.qb200_test_override(key, 0)
    assert family == 1
    # oracle, bit-exact, on two rows of every 32-row band (all columns)
    rows = band_rows(M, seed=N + 1)
    ref = O.to_f32(O.qbytes_int_mm(A[rows], W, s, tag), tag)
    if bias is not None:
        ref = O.round_to(ref + bias, tag)
    got = torch_to_bits(y[torch.from_numpy(rows).cuda()])
    assert np.array_equal(got, O.from_f32(ref, tag)), (variant, N)
    # every element, bit-exact, against the same arithmetic on the device
    acc = _int_product_on_device(At, Wt)
    full = (acc.float() * st.float().reshape(1, -1)).to(torch.bfloat16)
    if bt is not None:
        full = (full + bt).to(torch.bfloat16)
    assert torch.equal(y, full), (variant, N, int((y != full).sum()))


@pytest.mark.parametrize("N", [4096, 14336])
def test_fp8_bench_shapes(N):
    M, K, tag, akind, wkind = 4096, 4096, "bf16", "e4m3fn", "e4m3fn"
    rng = np.random.default_rng(N + 5)
    a_bits = O.f32_to_fp8_bits(np.clip(rng.standard_normal((M, K), dtype=np.float32), -3, 3), akind)
    w_bits = O.f32_to_fp8_bits(np.clip(rng.standard_normal((N, K), dtype=np.float32) * 2, -6, 6), wkind)
    s = O.round_to(rng.random(N, dtype=np.float32) / 1e2 + 1e-4, tag)
    At, Wt, st = bits_to_torch(a_bits, akind), bits_to_torch(w_bits, wkind), bits_to_torch(O.from_f32(s, tag), tag)
    y, family = cabi_qbytes_mm(At, Wt, st)
    torch.cuda.synchronize()
    assert family == 1
    rows = band_rows(M, seed=N + 2)
    y64, _ = O.qbytes_mm_fp8_native(a_bits[rows], akind, w_bits, wkind, s, tag)
    a, w = O.fp8_bits_to_f32(a_bits[rows], akind), O.fp8_bits_to_f32(w_bits, wkind)
    bound = 0.51 * O.ulp(y64, tag) + O.accumulate_allowance(a, w) * s.reshape(1, -1)
    yg = torch_to_f32(y[torch.from_numpy(rows).cuda()]).astype(np.float64)
    assert np.all(np.abs(yg - y64) <= bound), float(np.max(np.abs(yg - y64) / bound))
    # every element against the fp32 product of the same operands on the device
    full = (torch.matmul(At.float(), Wt.float().t()) * st.float().reshape(1, -1)).to(torch.bfloat16)
    d = y.float() - full.float()
    assert float(d.norm() / full.float().norm()) < 1e-3
    assert int((d.abs() > full.float().abs() * 2.0 ** -6 + 2.0 ** -6 * full.float().abs().mean()).sum()) == 0


@pytest.mark.parametrize("wkind", ["int8", "e4m3fn"])
def test_weight_only_bench_shape(wkind):
    """bf16 activations x int8 / fp8 weights at (4096, 14336, 4096): operands rnd(scale * W) as the reference builds them
    (library/qbytes_mm.py:25-33), persistent loop of 7 tiles per CTA."""
    M, N, K, tag = 4096, 14336, 4096, "bf16"
    rng = np.random.default_rng(3)
    a = O.round_to(rng.standard_normal((M, K), dtype=np.float32), tag)
    if wkind == "int8":
        w_store = rng.integers(-128, 128, size=(N, K), dtype=np.int8)
        w = w_store.astype(np.float32)
    else:
        w_store = O.f32_to_fp8_bits(np.clip(rng.standard_normal((N, K), dtype=np.float32) * 3, -200, 200), wkind)
        w = O.fp8_bits_to_f32(w_store, wkind)
    s = O.round_to(rng.random(N, dtype=np.float32) / 1e2 + 1e-4, tag)
    At, Wt, st = bits_to_torch(O.from_f32(a, tag), tag), bits_to_torch(w_store, wkind), bits_to_torch(O.from_f32(s, tag), tag)
    y, family = cabi_qbytes_mm(At, Wt, st)
    torch.cuda.synchronize()
    assert family == 1
    rows = band_rows(M, seed=9)
    ap, wp = O.qbytes_mm_operands(a[rows], w, s, tag)
    y64, _, tol = O.linear_from_dequantized(ap, wp, None, tag)
    bound = 1.02 * tol + O.accumulate_allowance(ap, wp)
    err = np.abs(torch_to_f32(y[torch.from_numpy(rows).cuda()]).astype(np.float64) - y64)
    assert np.all(err <= bound), (wkind, float(np.max(err / bound)))
    ws_t = (st.reshape(-1, 1) * Wt.to(torch.bfloat16)).to(torch.bfloat16)  # the reference's operand, on the device
    check_full_against_device_fp32(y, At, ws_t, None, ("weight_only", wkind))


# ------------------------------------------------------------------------------------------------- hardening
def test_second_device_in_one_process():
    """Function attributes, SM count and the architecture check are cached per DEVICE: a >48 KB-shared-memory kernel must
    launch on cuda:1 after it ran on cuda:0 (ADVICE r1: per-process statics broke this)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    M, N, K, tag = 256, 1024, 1024, "bf16"
    q, packed, scale, shift = make_qbits_weights(N, K, 128, tag, seed=1)
    rng = np.random.default_rng(0)
    x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
    outs = []
    for dev in ("cuda:0", "cuda:1", "cuda:0"):
        with torch.cuda.device(dev):
            y = cabi_qbits_mm(bits_to_torch(x_bits, tag, dev), torch.from_numpy(packed).to(dev), bits_to_torch(scale, tag, dev),
                              bits_to_torch(shift, tag, dev), None, N, K, 128)
            a = torch.randint(-127, 127, (M, K), dtype=torch.int8, device=dev)
            cabi_qbytes_mm(a, torch.randint(-127, 127, (N, K), dtype=torch.int8, device=dev),
                           torch.ones(N, dtype=torch.bfloat16, device=dev))
            torch.cuda.synchronize(dev)
            outs.append(y.cpu())
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


# ------------------------------------------------------------------------------------- fused all-gather, one GPU
@pytest.mark.parametrize("M", [1, 8, 40, 300, 4096])
@pytest.mark.parametrize("world", [2, 8])
def test_fused_gather_emulated_on_one_gpu(M, world):
    """The column-parallel kernels with the all-gather fused in (qb200_qbits_mm_gather), exercised on ONE device: the
    `world` "ranks" are `world` output buffers and flag arrays on the same GPU and the ranks' kernels run one after the
    other.  Checks the peer stores (every rank's slab lands in every buffer at its column offset, wgmma epilogue for
    M > 8, ring-gemv reducer for M <= 8), bit-identity with the single-rank linear on the full weight, and the flag
    protocol (epochs published to every flag array; a kernel that waits for its input passes once all ranks published)."""
    import ctypes
    from quanto_b200.parallel import shard_weight
    import quanto_b200 as q
    n = native()
    lib = n.load()
    N, K, G, tag = (14336 if M != 300 else 4096), 4096, 128, "bf16"
    if world == 8 and M == 300:
        pytest.skip("one shape per world size is enough for the mid-M kernel")
    _, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=world + M)
    rows_g = N * K // G
    w_full = q.WeightQBitsTensor(q.qint4, 0, G, torch.Size([N, K]), (K, 1),
                                 q.PackedTensor(torch.from_numpy(packed).cuda(), 4, torch.Size([rows_g, G]), (G, 1)),
                                 bits_to_torch(scale, tag).reshape(-1, 1), bits_to_torch(shift, tag).reshape(-1, 1))
    x = torch.randn(M, K, device="cuda").to(torch.bfloat16)
    # 8 < M <= 128 runs the stream-K kernel, whose split of K (and so the fp32 summation order) depends on the shard
    # shape: those outputs are compared within the accumulation-order tolerance instead of bit for bit
    exact = not (8 < M <= 128)
    y_ref = torch.nn.functional.linear(x, w_full)

    def same(b):
        if exact:
            return torch.equal(b, y_ref)
        d = (b.float() - y_ref.float()).abs()
        return bool(torch.isfinite(b.float()).all()) and float(d.max()) <= 2.0 ** -6 * float(y_ref.float().abs().max())
    n_local = N // world
    bufs = [torch.full((M, N), float("nan"), dtype=torch.bfloat16, device="cuda") for _ in range(world)]
    flags = [torch.zeros(64, dtype=torch.int32, device="cuda") for _ in range(world)]
    out_ptrs = (ctypes.c_void_p * world)(*[b.data_ptr() for b in bufs])
    flag_ptrs = (ctypes.c_void_p * world)(*[f.data_ptr() for f in flags])
    stream = n.stream_ptr(x.device)

    def launch(rank, wait_flags):
        w = shard_weight(w_full, rank, world)
        ws = n.workspace(x.device, stream, lib.qb200_qbits_mm_workspace_bytes(M, n_local, K))
        n.check(lib.qb200_qbits_mm_gather(x.data_ptr(), w._data._data.data_ptr(), w._scale.data_ptr(), w._shift.data_ptr(),
                                          None, out_ptrs, flag_ptrs, world, rank, wait_flags, M, n_local, K, G,
                                          n.DTYPE_CODE[x.dtype], 0, n.ptr(ws), 0 if ws is None else ws.numel(), stream),
                "qbits_mm_gather")
        return w

    keep = [launch(r, 0) for r in range(world)]
    torch.cuda.synchronize()
    for b in bufs:
        assert same(b)
    for r in range(world):
        f = flags[r].cpu()
        assert f[:world].tolist() == [1] * world and int(f[world]) == 1 and int(f[world + 1]) == 0, f[: world + 2].tolist()
    # second round: every kernel waits for its input (epoch 1 is already published everywhere) and, for the last rank,
    # for the output too (all other ranks have published epoch 2 by then)
    for b in bufs:
        b.fill_(float("nan"))
    for r in range(world):
        launch(r, n.GATHER_WAIT_INPUT | (n.GATHER_WAIT_OUTPUT if r == world - 1 else 0))
    torch.cuda.synchronize()
    for b in bufs:
        assert same(b)
    assert flags[0].cpu()[: world + 1].tolist() == [2] * (world + 1)
    del keep
