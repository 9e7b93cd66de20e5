"""Every shipped instantiation of the small-M (decode) int4 kernels, run at its edges against the float64 oracle.

Below M = 32 the int4 linear runs on three kernels of kernel family 3 (api_qbits_small.cu):
* gemv_w4r, the second-generation TMA-ring gemv (M <= 16): 68 instantiations, one census row each;
* gemv_w4s, the first-generation TMA-ring gemv (M <= 8): 8 instantiations (dtype x zero-point x coefficient ring);
* gemv_w4, the stream-K warp-MMA gemv (M <= 32 when forced): 12 instantiations (dtype x zero-point x token tile).
Each row forces its kernel, checks the whole output with helpers.check_linear and the run-to-run determinism.  Which
gemv_w4r instantiation a row reaches is read from the dispatcher's own plan (qb200_qbits_ring_plan, host only), so a row
whose shape stops landing on its instantiation fails on a machine without a GPU.  The last test checks on the device what
column-parallel decode relies on: a weight shard's output is bit-identical to the same columns of the full output.
"""
import contextlib
import ctypes
import itertools

import numpy as np
import pytest
import torch

from helpers import O, bits_to_torch, cabi_qbits_mm, check_linear, make_qbits_weights, native

SMS_H100 = 132  # the plan query's grid on a machine without a GPU (H100 SXM)
DECODE_TICKET_BYTES = 64 * 1024  # kDecodeTicketBytes: the stream-K ticket counters at the start of the workspace
LITE_SMEM = 112 * 1024  # the two-CTAs-per-SM ("lite") shape keeps each CTA under this


@contextlib.contextmanager
def _overrides(pairs):
    n = native()
    with contextlib.ExitStack() as stack:
        for key, value in pairs:
            stack.enter_context(n.test_override(getattr(n, key), value))
        yield


def _case(M, N, K, G, tag, zp, seed, unaligned=False, oracle=True):
    """Weights, activations and (odd M) a bias: the oracle's storage bits and the device arguments of cabi_qbits_mm.
    `unaligned`: the scales and shifts are views one element into a larger buffer (not 16-byte aligned).
    `oracle=False`: the device arguments only (no dequantised weight)."""
    _, packed, scale, shift = make_qbits_weights(N, K, G, tag, seed=seed, zeropoint=zp)
    rng = np.random.default_rng(seed + 1)
    x_bits = O.from_f32(rng.standard_normal((M, K), dtype=np.float32), tag)
    bias_bits = O.from_f32(rng.standard_normal(N, dtype=np.float32), tag) if M % 2 == 1 else None
    deq_bits = O.dequantize_qbits(packed, 4, scale, shift, tag, N, K, G, shift_is_int=zp) if oracle else None
    scale_t = bits_to_torch(scale, tag)
    shift_t = torch.from_numpy(shift).cuda() if zp else bits_to_torch(shift, tag)
    if unaligned:
        scale_t = torch.cat([scale_t[:1], scale_t])[1:]
        shift_t = torch.cat([shift_t[:1], shift_t])[1:]
        assert scale_t.data_ptr() % 16 != 0 and shift_t.data_ptr() % 16 != 0
    args = (bits_to_torch(x_bits, tag), torch.from_numpy(packed).cuda(), scale_t, shift_t,
            None if bias_bits is None else bits_to_torch(bias_bits, tag), N, K, G)
    return x_bits, deq_bits, bias_bits, args


def _sm_count():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


# ------------------------------------------------------------------------------------------ gemv_w4r census
# launch_gemvr / launch_gemvr_shape: per (dtype, zero-point), token groups TG 1 with (slabs per warp SPW, log2(group / 64)
# GL) in (4,1) (2,1) (4,0) (2,0) (1,0), one pass or several passes over K (MPASS); TG 2 with the same five, one pass; and
# the opt-in "lite" shape (two CTAs per SM, SPW 2) with GL 0 / 1.  17 per (dtype, zero-point), 68 in all.
# Shapes per instantiation, one per (dtype, zero-point) in the order bf16 / shift, bf16 / zp, f16 / shift, f16 / zp:
# (M, N, K, G).  Together they run M off a multiple of 8 (the last token aliases the padding rows), odd M with a bias,
# N / 16 below the grid (N = 144, 400), just above it (N = 2128: some CTAs own two row groups) and ragged row groups per
# CTA (N = 4112).  Multi-pass rows have one row group per CTA here; the shard test below runs them with two.
RING2_SHAPES = {
    # (TG, SPW, GL, MPASS, lite)
    (1, 4, 1, False, False): [(1, 144, 4096, 128), (3, 2128, 4096, 128), (6, 4112, 4096, 128), (8, 144, 4096, 128)],
    (1, 2, 1, False, False): [(2, 2128, 2048, 128), (5, 144, 2048, 128), (7, 144, 2048, 128), (3, 4112, 2048, 128)],
    (1, 4, 0, False, False): [(5, 4112, 4096, 64), (8, 144, 4096, 64), (1, 2128, 4096, 64), (6, 144, 4096, 64)],
    (1, 2, 0, False, False): [(3, 144, 2048, 64), (6, 4112, 2048, 64), (4, 144, 2048, 64), (1, 2128, 2048, 64)],
    (1, 1, 0, False, False): [(7, 144, 1024, 64), (1, 144, 1024, 64), (3, 2128, 3072, 64), (5, 4112, 3072, 64)],
    (1, 4, 1, True, False): [(8, 144, 8192, 128), (5, 144, 12288, 128), (6, 400, 12288, 128), (8, 400, 8192, 128)],
    (1, 2, 1, True, False): [(7, 144, 10240, 128), (6, 144, 14336, 128), (8, 400, 10240, 128), (5, 144, 14336, 128)],
    (1, 4, 0, True, False): [(7, 400, 8192, 64), (6, 144, 12288, 64), (8, 144, 8192, 64), (5, 144, 12288, 64)],
    (1, 2, 0, True, False): [(6, 144, 10240, 64), (7, 400, 10240, 64), (4, 144, 14336, 64), (8, 144, 10240, 64)],
    (1, 1, 0, True, False): [(7, 144, 9216, 64), (6, 144, 11264, 64), (8, 400, 11264, 64), (5, 144, 13312, 64)],
    (2, 4, 1, False, False): [(9, 144, 4096, 128), (11, 2128, 4096, 128), (12, 4112, 4096, 128), (10, 144, 4096, 128)],
    (2, 2, 1, False, False): [(14, 2128, 2048, 128), (16, 144, 4096, 128), (11, 144, 2048, 128), (13, 4112, 4096, 128)],
    (2, 4, 0, False, False): [(11, 4112, 4096, 64), (9, 144, 4096, 64), (10, 2128, 4096, 64), (11, 144, 4096, 64)],
    (2, 2, 0, False, False): [(12, 144, 4096, 64), (14, 144, 2048, 64), (15, 4112, 2048, 64), (16, 2128, 4096, 64)],
    (2, 1, 0, False, False): [(13, 144, 1024, 64), (10, 2128, 3072, 64), (16, 144, 3072, 64), (9, 4112, 1024, 64)],
    (1, 2, 1, False, True): [(1, 144, 4096, 128), (2, 2128, 2048, 128), (2, 144, 4096, 128), (1, 4112, 2048, 128)],
    (1, 2, 0, False, True): [(2, 144, 2048, 64), (1, 144, 4096, 64), (1, 2128, 4096, 64), (2, 4112, 2048, 64)],
}
TAG_ZP = list(itertools.product(("bf16", "f16"), (False, True)))


def _ring2_census():
    rows = []
    for j, (tag, zp) in enumerate(TAG_ZP):
        for (tg, spw, gl, mpass, lite), shapes in RING2_SHAPES.items():
            M, N, K, G = shapes[j]
            name = (f"{tag}-{'zp' if zp else 'shift'}-" + ("lite" if lite else f"tg{tg}") +
                    f"-spw{spw}-gl{gl}" + ("-mpass" if mpass else "") + f"-m{M}-n{N}-k{K}-g{G}")
            rows.append(dict(id=name, tag=tag, zp=zp, tg=tg, spw=spw, gl=gl, mpass=mpass, lite=lite, M=M, N=N, K=K, G=G))
    return rows


RING2 = _ring2_census()
assert len(RING2) == 68
assert len({(r["tag"], r["zp"], r["tg"], r["spw"], r["gl"], r["mpass"], r["lite"]) for r in RING2}) == 68
assert {144, 2128, 4112} <= {r["N"] for r in RING2}
assert any(r["M"] % 8 != 0 for r in RING2) and any(r["M"] % 2 == 1 for r in RING2)
assert all(r["K"] <= 4096 for r in RING2 if r["N"] > 400)  # the float64 oracle stays small


def _ring2_plan(M, N, K, G, zp, sms, lite):
    """(slabs per warp, passes over K, ring stages, token groups, shared memory bytes) of the dispatcher's plan, or None."""
    lib = native().load()
    out = (ctypes.c_int * 5)()
    with _overrides([("OVR_GEMV_SHAPE", 2)] if lite else []):
        ok = lib.qb200_qbits_ring_plan(M, N, K, G, int(zp), min(N // 16, sms), out)
    return tuple(out) if ok else None


def _assert_lands(row, sms):
    plan = _ring2_plan(row["M"], row["N"], row["K"], row["G"], row["zp"], sms, row["lite"])
    assert plan is not None, (row["id"], "the ring kernel does not take this shape")
    spw, passes, _, tg, smem = plan
    assert row["gl"] == (1 if row["G"] == 128 else 0)
    assert (spw, passes > 1, tg) == (row["spw"], row["mpass"], row["tg"]), (row["id"], plan)
    if row["lite"]:
        assert spw == 2 and passes == 1 and smem <= LITE_SMEM, (row["id"], plan)


@pytest.mark.parametrize("row", RING2, ids=[r["id"] for r in RING2])
def test_ring2_row_lands_on_its_instantiation(row):
    _assert_lands(row, SMS_H100)


@pytest.mark.gpu
@pytest.mark.parametrize("row", RING2, ids=[r["id"] for r in RING2])
def test_ring2_census(row):
    _assert_lands(row, _sm_count())
    M, N, K, G, tag, zp = row["M"], row["N"], row["K"], row["G"], row["tag"], row["zp"]
    x_bits, deq_bits, bias_bits, args = _case(M, N, K, G, tag, zp, seed=M + N + K + G + 7 * zp)
    lib = native().load()
    with _overrides([("OVR_INT4_ROUTE", native().ROUTE_INT4_RING2)] + ([("OVR_GEMV_SHAPE", 2)] if row["lite"] else [])):
        y1 = cabi_qbits_mm(*args)
        fam = lib.qb200_last_kernel_family()
        y2 = cabi_qbits_mm(*args)
        y3 = cabi_qbits_mm(*args, use_workspace=False)
        torch.cuda.synchronize()
    assert fam == 3
    assert torch.equal(y1, y2) and torch.equal(y1, y3)
    check_linear(y1, x_bits, deq_bits, bias_bits, tag, row["id"])
    y0 = cabi_qbits_mm(*args)  # the dispatcher's own choice passes the same bound
    torch.cuda.synchronize()
    check_linear(y0, x_bits, deq_bits, bias_bits, tag, ("auto", row["id"]))


# ------------------------------------------------------------------------------------------ gemv_w4s census
# launch_gemvs: per (dtype, zero-point), the coefficient ring (CR: scales / shifts as bulk copies) or LDG at first use.
# make_gemvs_plan takes the ring when a row group's scale run is 16-byte granular (K / G * 2 % 16 == 0; zero-points:
# K / G % 16 == 0) and the coefficients are 16-byte aligned.  (tag, zp, CR, M, N, K, G, unaligned coefficients); N / 2 is
# never a multiple of the grid (min(N / 2, SMs)), K = 11008 is cut into four chunks of 2752.
RING1 = [
    ("bf16", False, True, 1, 298, 4096, 128, False),
    ("bf16", False, False, 3, 1000, 11008, 128, False),
    ("bf16", True, True, 2, 2050, 2048, 128, False),
    ("bf16", True, False, 6, 530, 1024, 128, False),
    ("f16", False, True, 8, 1000, 1024, 32, False),
    ("f16", False, False, 5, 298, 4096, 64, True),
    ("f16", True, True, 4, 1000, 4096, 128, False),
    ("f16", True, False, 5, 530, 11008, 64, False),
]
RING1_IDS = [f"{t}-{'zp' if z else 'shift'}-{'cr' if c else 'ldg'}-m{m}-n{n}-k{k}-g{g}{'-unaligned' if u else ''}"
             for t, z, c, m, n, k, g, u in RING1]
assert len({r[:3] for r in RING1}) == 8
assert any(r[5] == 11008 for r in RING1) and any(r[6] == 32 for r in RING1) and any(r[7] for r in RING1)


@pytest.mark.parametrize("row", RING1, ids=RING1_IDS)
def test_ring1_row_selects_its_coefficient_path(row):
    tag, zp, cr, M, N, K, G, unaligned = row
    gpr = K // G
    assert cr == (not unaligned and gpr * 2 % 16 == 0 and (not zp or gpr % 16 == 0))
    assert 1 <= M <= 8 and (N // 2) % min(N // 2, SMS_H100) != 0


@pytest.mark.gpu
@pytest.mark.parametrize("row", RING1, ids=RING1_IDS)
def test_ring1_census(row):
    tag, zp, cr, M, N, K, G, unaligned = row
    x_bits, deq_bits, bias_bits, args = _case(M, N, K, G, tag, zp, seed=M + N + K + G, unaligned=unaligned)
    n = native()
    lib = n.load()
    with n.test_override(n.OVR_INT4_ROUTE, n.ROUTE_INT4_RING):
        y1 = cabi_qbits_mm(*args)
        fam = lib.qb200_last_kernel_family()
        y2 = cabi_qbits_mm(*args, use_workspace=False)
        torch.cuda.synchronize()
        assert fam == 3
        assert torch.equal(y1, y2)
        check_linear(y1, x_bits, deq_bits, bias_bits, tag, RING1_IDS[RING1.index(row)])
        if (K, zp) == (11008, False):  # multi-chunk K: the same bits whichever lanes issue the copies
            for pmode in (1, 2, 3):
                with n.test_override(n.OVR_GEMV_PRODUCER, pmode):
                    yp = cabi_qbits_mm(*args)
                    torch.cuda.synchronize()
                assert torch.equal(y1, yp), pmode


# ------------------------------------------------------------------------------------------ gemv_w4 census
# launch_gemv_mt: per (dtype, zero-point), token tiles MT 1 / 2 / 4 for M <= 8 / <= 16 / <= 32.  (tag, zp, M, N, K, G):
# N / 2 % 64 != 0 leaves a partial out-feature block, K = 128 is a single 128-k stage, K = 14336 many segments per block.
GEMV = [
    ("bf16", False, 1, 200, 128, 64), ("bf16", False, 13, 1000, 4096, 128), ("bf16", False, 32, 520, 14336, 128),
    ("bf16", True, 7, 1000, 14336, 128), ("bf16", True, 9, 200, 128, 128), ("bf16", True, 19, 1000, 4096, 32),
    ("f16", False, 8, 4096, 4096, 64), ("f16", False, 16, 1000, 14336, 64), ("f16", False, 17, 200, 128, 128),
    ("f16", True, 3, 1000, 4096, 128), ("f16", True, 11, 2064, 14336, 128), ("f16", True, 25, 1000, 128, 64),
]


def _mt(M):
    return 1 if M <= 8 else 2 if M <= 16 else 4


GEMV_IDS = [f"{t}-{'zp' if z else 'shift'}-mt{_mt(m)}-m{m}-n{n}-k{k}-g{g}" for t, z, m, n, k, g in GEMV]
assert len({(t, z, _mt(m)) for t, z, m, *_ in GEMV}) == 12
assert {128, 14336} <= {r[4] for r in GEMV} and any((r[3] // 2) % 64 != 0 for r in GEMV)


@pytest.mark.parametrize("row", GEMV, ids=GEMV_IDS)
def test_gemv_row_takes_the_warp_mma_kernel(row):
    """Shapes the stream-K kernel takes (decode_applicable): N even, K % 128 == 0, G % 16 == 0, M <= 32."""
    tag, zp, M, N, K, G = row
    assert 1 <= M <= 32 and N % 2 == 0 and K % 128 == 0 and G % 16 == 0 and K % G == 0


def _gemv_run(args):
    n = native()
    with n.test_override(n.OVR_INT4_ROUTE, n.ROUTE_INT4_GEMV):
        y = cabi_qbits_mm(*args)
        fam = n.load().qb200_last_kernel_family()
    assert fam == 3
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("row", GEMV, ids=GEMV_IDS)
def test_gemv_census(row):
    tag, zp, M, N, K, G = row
    x_bits, deq_bits, bias_bits, args = _case(M, N, K, G, tag, zp, seed=M + N + K + G)
    y1 = _gemv_run(args)
    y2 = _gemv_run(args)
    torch.cuda.synchronize()
    assert torch.equal(y1, y2)  # deterministic split-K reduction
    check_linear(y1, x_bits, deq_bits, bias_bits, tag, GEMV_IDS[GEMV.index(row)])


@pytest.mark.gpu
def test_gemv_leaves_its_tickets_zero():
    """The 12 instantiations back to back on one stream share one workspace; each must hand its ticket counters back
    zeroed (the buffer is zeroed only when allocated), so the next shape's fix-up starts from zero."""
    n = native()
    lib = n.load()
    dev = torch.device("cuda", torch.cuda.current_device())
    stream = n.stream_ptr(dev)
    ws = n.workspace(dev, stream, max(lib.qb200_qbits_mm_workspace_bytes(m, nn, k) for _, _, m, nn, k, _ in GEMV))
    cases = [_case(M, N, K, G, tag, zp, seed=M + N + K + G, oracle=False)[3] for tag, zp, M, N, K, G in GEMV]
    first = _gemv_run(cases[0])
    for args in cases[1:]:
        _gemv_run(args)
    torch.cuda.synchronize()
    assert n.workspace(dev, stream, 1) is ws  # every launch used this buffer
    nonzero = int(torch.count_nonzero(ws[:DECODE_TICKET_BYTES]))
    assert nonzero == 0, nonzero
    again = _gemv_run(cases[0])
    torch.cuda.synchronize()
    assert torch.equal(first, again)


# ------------------------------------------------------------------------------------------ shard bit-identity
# Column-parallel decode: rank r of P computes out-features [r N / P, (r + 1) N / P) from its own slice of the packed
# rows, scales and shifts, and must reproduce those columns of the full output bit for bit.  The plan cuts K the same way
# for both (test_host_logic); here the device runs it, one and several passes, one and two row groups per CTA.
SHARD_N = 4096
SHARD_M = (1, 2, 5, 8, 12, 16)
SHARD_WORLDS = (2, 4, 8)


def _pack_rows(q):
    """[N, K] nibbles -> the canonical packed [N / 2, K] bytes: out-feature n in the low nibble of packed row n, out-feature
    n + N / 2 in the high nibble (pack_weights on the [N * K / G, G] grouped weight)."""
    h = q.shape[0] // 2
    return q[:h] | (q[h:] << 4)


@pytest.mark.gpu
@pytest.mark.parametrize("zp", [False, True], ids=["shift", "zp"])
@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("K,G", [(4096, 128), (14336, 128), (11264, 64)])
def test_ring2_shard_is_bit_identical_to_the_full_output(K, G, tag, zp):
    n = native()
    dt = {"bf16": torch.bfloat16, "f16": torch.float16}[tag]
    gen = torch.Generator(device="cuda").manual_seed(K + G + 2 * zp)
    N, gpr = SHARD_N, K // G
    q = torch.randint(0, 16, (N, K), dtype=torch.uint8, device="cuda", generator=gen)
    scale = (torch.rand(N * gpr, device="cuda", generator=gen) * 0.01 + 0.002).to(dt)
    if zp:
        shift = torch.randint(0, 16, (N * gpr,), dtype=torch.uint8, device="cuda", generator=gen)
    else:
        shift = (scale.float() * (7 + 2 * torch.rand(N * gpr, device="cuda", generator=gen))).to(dt)
    bias = torch.randn(N, device="cuda", generator=gen).to(dt)
    packed = _pack_rows(q)
    sms = _sm_count()
    ran = 0
    for M in SHARD_M:
        full_plan = _ring2_plan(M, N, K, G, zp, sms, False)
        # the activations of M > 8 tokens do not fit shared memory at these K, and several passes are for M <= 8 only
        assert (full_plan is not None) == (M <= 8 or K == 4096), (M, full_plan)
        if full_plan is None:
            continue
        if (M, K) == (8, 14336):
            assert full_plan[1] == 7, full_plan
        x = torch.randn(M, K, device="cuda", generator=gen).to(dt)
        b = bias if M % 2 else None
        with n.test_override(n.OVR_INT4_ROUTE, n.ROUTE_INT4_RING2):
            full = cabi_qbits_mm(x, packed, scale, shift, b, N, K, G)
            for P in SHARD_WORLDS:
                ns = N // P
                shard_plan = _ring2_plan(M, ns, K, G, zp, sms, False)
                assert shard_plan is not None and shard_plan[:2] == full_plan[:2] and shard_plan[3] == full_plan[3]
                for r in range(P):
                    lo, hi = r * ns, (r + 1) * ns
                    y = cabi_qbits_mm(x, _pack_rows(q[lo:hi]), scale[lo * gpr:hi * gpr], shift[lo * gpr:hi * gpr],
                                      None if b is None else b[lo:hi], ns, K, G)
                    torch.cuda.synchronize()
                    assert torch.equal(full[:, lo:hi], y), (M, P, r)
                    ran += 1
    assert ran == sum(2 + 4 + 8 for M in SHARD_M if M <= 8 or K == 4096)
