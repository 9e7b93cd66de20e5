"""The HQQ optimizer restated on the numpy oracle (oracle/quanto_oracle.py), with exact sums.

TEST INFRASTRUCTURE ONLY, like quanto_oracle.py.  Pinned by tests/test_hqq_oracle.py against tests/golden/hqq.npz,
which oracle/gen_golden_hqq.py produces from the real reference.  Follows
optimum/quanto/tensor/optimizers/hqq_optimizer.py:28-34 (shrink_lp_op) and :60-87 (optimize), on the CPU arithmetic
of torch for bf16 / fp16 tensors:
  * torch.pow(t, lp - 1) uses the exponent rounded to the tensor dtype and equals the float32 power rounded to the
    dtype: round_dt(round_f32(pow_f64(|x|, e_dt))) on every pattern (rounding pow_f64 straight to the dtype differs on
    one magnitude per dtype, where the float64 power lies within 2^-24 of a dtype midpoint);
  * (1.0 / beta) * t multiplies by the fp32 scalar and rounds once; |x| - 1.0 / beta subtracts the scalar rounded to
    the tensor dtype (lp_norm == 1);
  * torch.sign(NaN) == 0 and torch.sign(+-0) == +0;
  * torch.mean rounds once: round_dt(sum / n) with the sum taken in float64.
"""
import numpy as np

from . import quanto_oracle as O


def round64(x: np.ndarray, tag: str) -> np.ndarray:
    """float64 -> `tag` with ONE round-to-nearest-even (no detour through float32); returned as float32."""
    x = np.asarray(x, np.float64)
    if tag == "f16":
        with np.errstate(over="ignore"):
            return x.astype(np.float16).astype(np.float32)
    if tag != "bf16":
        raise ValueError(tag)
    with np.errstate(over="ignore", invalid="ignore"):
        m, e = np.frexp(x)  # x = m * 2^e, 0.5 <= |m| < 1
        e = np.maximum(e, -125)  # below 2^-126 the bf16 quantum is fixed at 2^-133
        r = np.ldexp(np.rint(np.ldexp(x, 8 - e)), e - 8)
        r = np.where(np.isfinite(x), r, x)
        r = np.where(np.abs(r) >= 2.0 ** 128, np.copysign(np.inf, x), r)
    return r.astype(np.float32)


def pow_exponent(lp_norm: float, tag: str) -> float:
    """The exponent torch.pow applies: python's lp_norm - 1 as a scalar of the tensor dtype."""
    return float(O.round_to(np.array([lp_norm - 1.0], np.float32), tag)[0])


def lp_pow(a_f32: np.ndarray, lp_norm: float, tag: str) -> np.ndarray:
    """torch.pow(|x|, lp_norm - 1) of a bf16 / fp16 tensor: round_dt(round_f32(pow_f64(|x|, e_dt)))."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        p = np.power(np.asarray(a_f32, np.float64), pow_exponent(lp_norm, tag)).astype(np.float32)
    return O.round_to(p, tag)


def shrink_lp(x_f32: np.ndarray, tag: str, beta: float, lp_norm: float) -> np.ndarray:
    """shrink_lp_op (hqq_optimizer.py:28-34) on values of `tag`; float32 values of `tag`."""
    x = np.asarray(x_f32, np.float32)
    a = np.abs(x)
    with np.errstate(invalid="ignore", over="ignore"):
        if lp_norm == 1:
            d = O.round_to(a - O.round_to(np.array([np.float32(1.0 / beta)]), tag)[0], tag)
        else:
            d = O.round_to(a - O.round_to(np.float32(1.0 / beta) * lp_pow(a, lp_norm, tag), tag), tag)
        r = np.where(d > 0, d, np.where(np.isnan(d), d, np.float32(0)))  # relu keeps NaN
        sgn = (x > 0).astype(np.float32) - (x < 0).astype(np.float32)  # torch.sign: NaN -> 0, +-0 -> +0
        return (sgn * r).astype(np.float32)


def _dequant(u, s, z, tag):
    """QBitsDequantizer with a float shift (quanto_oracle.dequantize_qbits): rnd(rnd(u * s) - z)."""
    return O.round_to(O.round_to(u * s, tag) - z, tag)


def _mean_abs(base, deq, tag) -> float:
    with np.errstate(invalid="ignore"):
        err = np.abs(O.round_to(base - deq, tag)).astype(np.float64)
    return float(round64(np.array([err.sum() / err.size]), tag)[0])


def hqq(grouped_f32: np.ndarray, tag: str, bits: int, lp_norm: float = 0.7, beta: float = 1e1, kappa: float = 1.01,
        iters: int = 20, zeropoint: bool = False, trajectory: bool = False):
    """HqqOptimizer()(W, qtype, axis=0, group_size) on an axis-0 grouped weight [R, G] (hqq_optimizer.py:60-87 after
    MaxOptimizer, affine_optimizer.py:52-63).

    Returns (scale storage [R,1], shift storage [R,1] or uint8 zero-points, errors, accepted): `errors` are the
    dt-rounded tensor-wide mean errors the loop computed (the start error, then one per iteration run, the last one the
    rejected iteration unless all `iters` were accepted), `accepted` the number of accepted iterations.  With
    `trajectory`, `errors` instead holds all iters + 1 means of the all-accepted trajectory, as the fused op reports them.
    """
    b = np.asarray(grouped_f32, np.float32)
    G = b.shape[1]
    scale_bits, shift_bits = O.max_optimizer(b, tag, bits)
    s = O.to_f32(scale_bits, tag)
    shift = O.to_f32(shift_bits, tag)
    u = O.quantize_affine(b, tag, bits, s, shift).astype(np.float32)
    errors = [_mean_abs(b, _dequant(u, s, shift, tag), tag)]
    best, accepted, stopped = errors[0], 0, False
    z = shift
    for i in range(iters):
        if stopped and not trajectory:
            break
        x = O.round_to(b - _dequant(u, s, z, tag), tag)
        e = shrink_lp(x, tag, beta, lp_norm)
        with np.errstate(invalid="ignore"):
            t = O.round_to(O.round_to(u * s, tag) - O.round_to(b - e, tag), tag)
        cand = round64(t.astype(np.float64).sum(axis=1, keepdims=True) / G, tag)
        u, z = O.quantize_affine(b, tag, bits, s, cand).astype(np.float32), cand
        err = _mean_abs(b, _dequant(u, s, z, tag), tag)
        errors.append(err)
        beta *= kappa  # only an accepted iteration reaches the next one: the all-accepted trajectory
        if stopped:
            continue
        if err < best:
            best, shift, accepted = err, cand, accepted + 1
        else:
            stopped = True
    if iters == 0 and not trajectory:
        errors = []  # the reference measures the start error inside its loop
    if zeropoint:
        with np.errstate(divide="ignore", invalid="ignore"):
            zp = np.clip(np.rint(O.round_to(shift / s, tag)), 0, 2 ** bits - 1)
        zp = np.where(np.isnan(zp), 0, zp).astype(np.uint8)  # the reference's NaN -> uint8 cast yields 0 on x86
        return scale_bits, zp, errors, accepted
    return scale_bits, O.from_f32(shift, tag), errors, accepted


def quantize_packed(grouped_f32, tag, bits, scale_bits, shift, zeropoint):
    """quantize_affine + pack_weights of the frozen layer with the HQQ scale / shift (canonical packed bytes)."""
    s = O.to_f32(scale_bits, tag)
    if zeropoint:
        data = O.quantize_affine(grouped_f32, tag, bits, s, shift, shift_is_int=True)
    else:
        data = O.quantize_affine(grouped_f32, tag, bits, s, O.to_f32(shift, tag))
    return O.pack_weights(data, bits)
