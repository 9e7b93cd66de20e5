"""CPU restatement (numpy) of the arithmetic shortcuts the quantisation kernels take (csrc/quantize_math.cuh,
csrc/freeze.cu), checked against the oracle.  The kernels must be bit-exact with the reference's op-by-op rounding, but
do not execute it literally: they multiply by a reciprocal instead of dividing, round through a magic-number addition
instead of cvt instructions, and (bf16) stay in packed 16-bit arithmetic.  Each identity used is pinned here, without a
GPU; an earlier draft of the zero-point path (zero-point folded into the rounding constant) failed exactly this check
before it ever ran on a GPU.
"""
import numpy as np

from oracle import quanto_oracle as O


def bf(x):
    return O.round_to(np.asarray(x, np.float32), "bf16")


def bf_bits(x):
    return O.from_f32(np.asarray(x, np.float32), "bf16").astype(np.uint32)


def test_reciprocal_multiply_equals_division_for_every_bf16_range():
    """scale = rnd(d / qmax): rnd_bf16(d * rcp(qmax)) is the same bf16 for EVERY positive normal bf16 d (qmax 15, 3, 127)."""
    d = O.bf16_bits_to_f32(np.arange(0x0080, 0x7F80, dtype=np.uint16))
    for qmax in (15.0, 3.0, 127.0):
        r = np.float32(1.0) / np.float32(qmax)  # correctly rounded, like rcp.rn / a folded constant
        fast = O.from_f32((d * r).astype(np.float32), "bf16")
        exact = O.from_f32((d / np.float32(qmax)).astype(np.float32), "bf16")
        assert np.array_equal(fast, exact), qmax


def test_reciprocal_multiply_equals_division_for_bf16_quotients():
    """t = rnd(x / s) for bf16 x, s: a quotient of two 8-bit significands is never closer than 2^-17 (relative) to a bf16
    rounding boundary unless it is exactly representable, so the 2^-22 error of x * rcp(s) cannot flip the rounding."""
    rng = np.random.default_rng(0)
    # all significand pairs at one exponent (the property is scale-invariant) + random exponents
    a = O.bf16_bits_to_f32((0x3F80 + np.arange(128, dtype=np.uint16))[:, None] + np.zeros((1, 128), np.uint16))
    s = O.bf16_bits_to_f32((0x3F80 + np.arange(128, dtype=np.uint16))[None, :] + np.zeros((128, 1), np.uint16))
    for ea in (-20, -3, 0, 5, 30):
        for es in (-25, -7, 0, 9):
            x = (a * np.float32(2.0**ea)).astype(np.float32)
            y = (s * np.float32(2.0**es)).astype(np.float32)
            r = (np.float32(1.0) / y).astype(np.float32)
            assert np.array_equal(bf_bits((x * r).astype(np.float32)), bf_bits((x / y).astype(np.float32))), (ea, es)
    x = bf(rng.standard_normal(200000).astype(np.float32) * 10.0 ** rng.uniform(-6, 6, 200000))
    y = bf(np.abs(rng.standard_normal(200000)).astype(np.float32) * 10.0 ** rng.uniform(-6, 6, 200000) + 1e-20)
    r = (np.float32(1.0) / y).astype(np.float32)
    assert np.array_equal(bf_bits((x * r).astype(np.float32)), bf_bits((x / y).astype(np.float32)))


def test_magic_add_is_rint_with_ties_to_even():
    """fp32: (t + 1.5 * 2^23) has bit pattern 0x4B400000 + rint(t) for |t| <= 2^22 (quantize_math.cuh rint_bits);
    bf16: (t + 192) has mantissa 64 + rint(t) for |t| <= 63 (the packed path of the fused freeze kernel)."""
    t = np.concatenate([np.arange(-300, 300, 0.25, dtype=np.float32), np.float32([127.5, -128.5, 2.5, 3.5, -0.5, 0.5]),
                        np.random.default_rng(1).uniform(-4e6, 4e6, 10000).astype(np.float32)])
    got = (t + np.float32(12582912.0)).astype(np.float32).view(np.int32) - 0x4B400000
    assert np.array_equal(got, np.rint(t).astype(np.int32))
    tb = bf(np.arange(-20, 20, 0.125, dtype=np.float32))  # includes every tie k + 0.5
    got_b = (bf_bits(bf(tb + np.float32(192.0))) & 0x7F).astype(np.int64) - 64
    assert np.array_equal(got_b, np.rint(tb).astype(np.int64))


def test_native_bf16_add_has_no_double_rounding():
    """b + z in one bf16 add (exact sum, one rounding) == the reference's fp32 add followed by a bf16 rounding."""
    rng = np.random.default_rng(2)
    a = bf(rng.standard_normal(300000).astype(np.float32) * 10.0 ** rng.uniform(-8, 8, 300000))
    b = bf(rng.standard_normal(300000).astype(np.float32) * 10.0 ** rng.uniform(-8, 8, 300000))
    two_step = bf_bits((a + b).astype(np.float32))  # fp32 add (rounded to 24 bits), then to bf16
    # f64 holds the exact sum of two bf16 numbers whenever their exponents differ by < 45; restrict to those
    ok = np.abs(np.log2(np.abs(a) + 1e-300) - np.log2(np.abs(b) + 1e-300)) < 40
    exact = a.astype(np.float64) + b.astype(np.float64)
    direct = O.from_f32(_round_f64_to_bf16(exact), "bf16").astype(np.uint32)
    assert ok.sum() > 200000 and np.array_equal(two_step[ok], direct[ok])


def _round_f64_to_bf16(x64):
    """Round float64 values to bf16 precision with ONE rounding (nearest even), returned as float32."""
    m, e = np.frexp(x64)  # x = m * 2^e, 0.5 <= |m| < 1
    scaled = np.ldexp(m, 8)  # 8 significant bits
    r = np.rint(scaled)  # ties to even
    return np.ldexp(r, e - 8).astype(np.float32)


def _emulate_packed_freeze(w, bits, zeropoint):
    """The bf16 fast path of quantize_qbits_max_kernel, statement by statement."""
    qmax = 2**bits - 1
    lo = w.min(axis=1, keepdims=True)
    hi = w.max(axis=1, keepdims=True)
    d = bf(hi - lo)
    with np.errstate(all="ignore"):
        s = np.where(d > 1e-30, bf((d * (np.float32(1.0) / np.float32(qmax))).astype(np.float32)), bf(d / np.float32(qmax)))
        fast = (np.abs(s) > 1e-30) & (np.abs(s) < 1e30)
        r = (np.float32(1.0) / s).astype(np.float32)
        z = -lo
        if zeropoint:
            zq = np.where(fast, bf((z * r).astype(np.float32)), bf(z / s))
            z = np.clip(np.rint(zq), 0, qmax)
            z = np.where(np.isnan(z), 0, z).astype(np.float32)
        a = w if zeropoint else bf(w + z)
        t = bf((a * r).astype(np.float32))
        cl_lo = -z if zeropoint else np.zeros_like(z)
        cl_hi = (qmax - z) if zeropoint else np.full_like(z, qmax)
        tc = np.minimum(np.maximum(t, cl_lo), cl_hi)
        tc = np.where(np.isnan(t), cl_lo, tc)  # hmax2 / hmin2 return the non-NaN operand
        m = bf(tc + np.float32(192.0))
        n = (bf_bits(m) & 0x7F).astype(np.int64) - (64 - (z.astype(np.int64) if zeropoint else 0))
    return s, z, n, fast


def test_packed_bf16_freeze_path_equals_the_oracle():
    rng = np.random.default_rng(3)
    for trial in range(60):
        spread = 10.0 ** rng.uniform(-7, 4)
        w = bf(rng.standard_normal((64, 128)).astype(np.float32) * spread + rng.uniform(-1, 1) * spread)
        if trial % 5 == 0:
            w = bf(np.round(w * 8) / 8)  # many exact ties
        for bits in (4, 2):
            for zeropoint in (False, True):
                s_ref, z_ref = O.max_optimizer(w, "bf16", bits, zeropoint)
                s, z, n, fast = _emulate_packed_freeze(w, bits, zeropoint)
                assert np.array_equal(O.from_f32(s, "bf16").reshape(-1), s_ref.reshape(-1))
                zr = z_ref.reshape(-1, 1) if zeropoint else O.to_f32(z_ref, "bf16").reshape(-1, 1)
                if zeropoint:
                    assert np.array_equal(z.reshape(-1).astype(np.uint8), z_ref.reshape(-1))
                ref = O.quantize_affine(w, "bf16", bits, O.to_f32(s_ref, "bf16").reshape(-1, 1), zr, zeropoint)
                sel = np.broadcast_to(fast, ref.shape)
                if not sel.any():
                    continue  # every scale outside the reciprocal's safe range: the kernel takes the IEEE division
                assert np.array_equal(n[sel], ref[sel].astype(np.int64)), (trial, bits, zeropoint)
                assert n[sel].min() >= 0 and n[sel].max() <= 2**bits - 1


def test_int8_magic_rounding_path_equals_the_oracle():
    """quantize_symmetric int8 (bf16 fast path): rnd(x * rcp(s)) -> NaN->0 -> clamp -> magic add -> low byte."""
    rng = np.random.default_rng(4)
    x = bf(rng.standard_normal((64, 512)).astype(np.float32) * 3)
    x[3] = 0  # an all-zero row: scale 0, quotient 0/0
    for per_row in (True, False):
        s_bits = O.absmax_scale(x, "bf16", 127.0, per_row)
        s = O.to_f32(s_bits, "bf16").reshape(-1, 1) if per_row else O.to_f32(s_bits, "bf16").reshape(1, 1)
        ref = O.quantize_symmetric(x, "bf16", "int8", s)
        with np.errstate(all="ignore"):
            fast = (np.abs(s) > 1e-30) & (np.abs(s) < 1e30)
            t = np.where(fast, bf((x * (np.float32(1.0) / s)).astype(np.float32)), bf(x / s))
            c = np.where(np.isnan(t), np.float32(0), t)
            c = np.minimum(np.maximum(c, np.float32(-128)), np.float32(127))
            q = ((c + np.float32(12582912.0)).astype(np.float32).view(np.int32) & 0xFF).astype(np.uint8).view(np.int8)
        assert np.array_equal(q, ref)


# ------------------------------------------------------------------------------------------- float8_e4m3fnuz
def _emulate_fnuz_encode(t):
    """quantize_one<DT_E4M3FNUZ> (csrc/quantize_math.cuh), statement by statement, on float32 quotients."""
    t = np.asarray(t, np.float32)
    with np.errstate(invalid="ignore"):
        c = np.minimum(np.maximum(np.where(np.isnan(t), np.float32(0), t), np.float32(-240)), np.float32(240))
    a = np.abs(c).astype(np.float32)
    # subnormal branch: rint_bits(a * 1024) through the 1.5 * 2^23 addition
    sub = ((a * np.float32(1024) + np.float32(12582912.0)).astype(np.float32).view(np.int32) - 0x4B400000).astype(np.uint32)
    u = a.view(np.uint32).astype(np.uint32)
    u = (u + np.uint32(0x7FFFF) + ((u >> 20) & 1)).astype(np.uint32)
    nrm = (((((u >> 23) & 0xFF) - 119) << 3) | ((u >> 20) & 7)).astype(np.uint32)
    b = np.where(a < np.float32(0.0078125), sub, nrm)
    out = np.where(b == 0, 0, b | np.where(c < 0, 0x80, 0)).astype(np.uint8)
    return np.where(np.isnan(t), np.uint8(0x80), out)


def test_fnuz_kernel_encoder_equals_the_oracle():
    """The hand-rolled RNE of the e4m3fnuz encoder == the oracle (pinned against torch's cast) for every finite bf16 and
    fp16 value, every tie / subnormal boundary in fp32, values past +-240, +-inf, NaN and +-0."""
    vals = [O.to_f32(np.arange(65536, dtype=np.uint16), tag) for tag in ("bf16", "f16")]
    mags = np.sort(O.fp8_bits_to_f32(np.arange(128, dtype=np.uint8), "e4m3fnuz").astype(np.float64))
    pts = np.concatenate([mags, (mags[:-1] + mags[1:]) / 2]).astype(np.float32)
    pts = np.concatenate([pts, np.nextafter(pts, np.float32(np.inf)), np.nextafter(pts, np.float32(-np.inf)),
                          np.float32([247.9, 248.0, 300.0, 3e38, np.inf, 2.0 ** -11, 1e-30, 0.0])])
    vals.append(np.concatenate([pts, -pts]))
    rng = np.random.default_rng(8)
    vals.append((rng.standard_normal(300000) * 10.0 ** rng.uniform(-5, 3, 300000)).astype(np.float32))
    for v in vals:
        v = v[~np.isnan(v)]
        ref = O.quantize_symmetric(v, "f32", "e4m3fnuz", np.float32(1.0))
        assert np.array_equal(_emulate_fnuz_encode(v), ref), int(np.sum(_emulate_fnuz_encode(v) != ref))
    assert _emulate_fnuz_encode(np.float32([np.nan, -0.0, -1e-6])).tolist() == [0x80, 0x00, 0x00]


def _emulate_fnuz_stage(codes, s_bits, tag):
    """cvt_bytes4<WT, 3> (csrc/gemm_tc.cuh): byte -> fp16 field pattern (bits << 7, sign to bit 15, the __vcmpeq2 patch
    turning 0x80 into a NaN), x 128 in fp16, then rnd_WT(scale * w) -- fp16 directly, bf16 via half -> float -> bf16."""
    t = np.asarray(codes, np.uint16)
    h = ((t & 0x7F) << 7) | ((t & 0x80) << 8)
    h = h | np.where(t == 0x80, 0x7FFF, 0).astype(np.uint16)
    w16 = (h.astype(np.uint16).view(np.float16) * np.float16(128)).astype(np.float16)
    if tag == "f16":
        s = s_bits.astype(np.uint16).view(np.float16)
        return (w16 * s).astype(np.float16).view(np.uint16)
    w = O.round_to(w16.astype(np.float32), "bf16")
    return O.from_f32((w * O.to_f32(s_bits, "bf16")).astype(np.float32), "bf16")


def _emulate_fnuz_to_float(codes):
    """e4m3fnuz_to_float (csrc/common.cuh), the decode of the CUDA-core qbytes_mm kernel."""
    t = np.asarray(codes, np.uint16)
    h = (((t & 0x7F) << 7) | ((t & 0x80) << 8)).astype(np.uint16)
    v = h.view(np.float16).astype(np.float32) * np.float32(128)
    return np.where(t == 0x80, np.float32(np.nan), v)


def test_fnuz_staging_decoder_equals_the_oracle():
    """Every one of the 256 codes times 2000 scales of each 16-bit type: the staged operand is the reference's
    rnd(scale * W.to(dtype)) bit for bit (NaN for 0x80), and the CUDA-core decode is the oracle's table."""
    codes = np.arange(256, dtype=np.uint8)
    w = O.fp8_bits_to_f32(codes, "e4m3fnuz")
    got = _emulate_fnuz_to_float(codes)
    assert np.array_equal(np.isnan(got), np.isnan(w)) and np.array_equal(got[~np.isnan(w)], w[~np.isnan(w)])
    rng = np.random.default_rng(9)
    for tag in ("f16", "bf16"):
        s = O.from_f32((10.0 ** rng.uniform(-7, 2, 2000)).astype(np.float32) * rng.choice([-1, 1], 2000), tag)
        s = np.concatenate([s, O.from_f32(np.float32([1.0, 2.0 ** -20, 0.0]), tag)])
        with np.errstate(over="ignore", invalid="ignore"):
            got = _emulate_fnuz_stage(codes[None, :], s[:, None], tag)
            ref = O.from_f32(O.to_f32(s, tag)[:, None] * O.round_to(w, tag)[None, :], tag)
        gnan, rnan = np.isnan(O.to_f32(got, tag)), np.isnan(O.to_f32(ref, tag))
        assert np.array_equal(gnan, rnan) and rnan[:, 0x80].all(), tag
        assert np.array_equal(got[~gnan], ref[~rnan]), (tag, int(np.sum(got[~gnan] != ref[~rnan])))
