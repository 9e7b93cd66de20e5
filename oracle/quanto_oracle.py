"""CPU oracle for the quantized-linear hot path of huggingface/optimum-quanto.

TEST INFRASTRUCTURE ONLY.  Nothing under ``optimum-quanto_b200/`` imports this
module; only ``tests/``, ``__graft_entry__.smoke()`` and the ``cpu_baseline`` /
``--impl reference`` legs of ``bench.py`` may.  The product path is CUDA-only.

This is a numpy restatement (no torch) of the reference arithmetic, written
from the reference's *behaviour*; each function cites the file:line it follows
(paths relative to the reference checkout, commit e33f8202).

Parity status: PINNED.  ``tests/test_oracle_golden.py`` checks every function
here against fixtures under ``tests/golden/`` that were produced by importing
the real reference in the authoring container (``oracle/gen_golden.py``).

Low-precision floats are carried as *bit patterns* (uint16 for bf16/fp16,
uint8 for fp8) next to a dtype tag, so that all comparisons are bit-exact and
independent of any framework's float formatting.
"""
from __future__ import annotations

import numpy as np

# --------------------------------------------------------------------------
# dtype helpers: every low precision format <-> float32, RNE
# --------------------------------------------------------------------------
FLOAT_TAGS = ("f32", "f16", "bf16")
FP8_TAGS = ("e4m3fn", "e5m2", "e4m3fnuz")


def bf16_bits_to_f32(bits: np.ndarray) -> np.ndarray:
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def f32_to_bf16_bits(x: np.ndarray) -> np.ndarray:
    """float32 -> bf16 bit pattern, round-to-nearest-even (what torch does for .to(bfloat16))."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    nan = np.isnan(x)
    rounded = (u + (((u >> 16) & 1) + np.uint32(0x7FFF))) >> 16
    rounded = np.where(nan, np.uint32(0x7FC0), rounded)
    return rounded.astype(np.uint16)


def f16_bits_to_f32(bits: np.ndarray) -> np.ndarray:
    return np.asarray(bits, dtype=np.uint16).view(np.float16).astype(np.float32)


def f32_to_f16_bits(x: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        return np.ascontiguousarray(x, dtype=np.float32).astype(np.float16).view(np.uint16)


def to_f32(bits_or_vals: np.ndarray, tag: str) -> np.ndarray:
    if tag == "f32":
        return np.asarray(bits_or_vals, dtype=np.float32)
    if tag == "bf16":
        return bf16_bits_to_f32(bits_or_vals)
    if tag == "f16":
        return f16_bits_to_f32(bits_or_vals)
    if tag in FP8_TAGS:
        return fp8_bits_to_f32(bits_or_vals, tag)
    raise ValueError(tag)


def from_f32(x: np.ndarray, tag: str) -> np.ndarray:
    """Round a float32 array to `tag` and return the storage representation."""
    if tag == "f32":
        return np.asarray(x, dtype=np.float32)
    if tag == "bf16":
        return f32_to_bf16_bits(x)
    if tag == "f16":
        return f32_to_f16_bits(x)
    if tag in FP8_TAGS:
        return f32_to_fp8_bits(x, tag)
    raise ValueError(tag)


def round_to(x: np.ndarray, tag: str) -> np.ndarray:
    """Round float32 values to the precision of `tag`, returned again as float32."""
    return to_f32(from_f32(x, tag), tag)


def _fp8_table(tag: str) -> np.ndarray:
    """Decode table for the 128 non-negative codes of an fp8 format (NaN/inf -> nan).

    e4m3fnuz (torch.float8_e4m3fnuz): bias 8, no infinities, all 128 codes finite; its only NaN is 0x80, the code
    that would be negative zero (see fp8_bits_to_f32).
    """
    if tag == "e4m3fn":
        ebits, mbits, bias = 4, 3, 7
    elif tag == "e5m2":
        ebits, mbits, bias = 5, 2, 15
    elif tag == "e4m3fnuz":
        ebits, mbits, bias = 4, 3, 8
    else:
        raise ValueError(tag)
    out = np.empty(128, dtype=np.float64)
    for code in range(128):
        e = code >> mbits
        m = code & ((1 << mbits) - 1)
        if e == 0:
            v = m * 2.0 ** (1 - bias - mbits)
        else:
            v = (1.0 + m * 2.0 ** (-mbits)) * 2.0 ** (e - bias)
        if tag == "e4m3fn" and code == 0x7F:
            v = np.nan
        if tag == "e5m2" and e == 31:
            v = np.inf if m == 0 else np.nan
        out[code] = v
    return out


_FP8_TABLES = {t: _fp8_table(t) for t in FP8_TAGS}
FP8_MAX = {"e4m3fn": 448.0, "e5m2": 57344.0, "e4m3fnuz": 240.0}


def fp8_bits_to_f32(bits: np.ndarray, tag: str) -> np.ndarray:
    b = np.asarray(bits, dtype=np.uint8)
    mag = _FP8_TABLES[tag][b & 0x7F]
    out = np.where(b & 0x80, -mag, mag)
    if tag == "e4m3fnuz":
        out = np.where(b == 0x80, np.nan, out)
    return out.astype(np.float32)


def f32_to_fp8_bits(x: np.ndarray, tag: str) -> np.ndarray:
    """RNE float32 -> fp8 for finite inputs with |x| <= finfo.max (callers clamp first).

    e4m3fnuz has no negative zero: a zero of either sign, and a negative value that rounds to zero, encode as 0x00;
    NaN encodes as 0x80 (torch's cast).
    """
    x = np.asarray(x, dtype=np.float32)
    table = _FP8_TABLES[tag]
    ncodes = int(np.sum(np.isfinite(table)))  # finite magnitudes are codes [0, ncodes)
    finite = table[:ncodes]
    a = np.abs(x).astype(np.float64)
    hi = np.searchsorted(finite, a, side="left")  # first code with value >= a
    hi = np.clip(hi, 0, ncodes - 1)
    lo = np.clip(hi - 1, 0, ncodes - 1)
    dlo = a - finite[lo]
    dhi = finite[hi] - a
    pick_hi = (dhi < dlo) | ((dhi == dlo) & ((hi & 1) == 0))
    code = np.where(pick_hi, hi, lo).astype(np.uint8)
    code = np.where(a == finite[hi], hi, code).astype(np.uint8)
    sign = (np.signbit(x)).astype(np.uint8) << 7
    if tag == "e4m3fnuz":
        sign = np.where(code == 0, np.uint8(0), sign)
        return np.where(np.isnan(x), np.uint8(0x80), code | sign).astype(np.uint8)
    code = np.where(np.isnan(x), np.uint8(0x7F), code)  # torch keeps NaN (0/0 of an all-zero row) as the NaN code
    return (code | sign).astype(np.uint8)


# --------------------------------------------------------------------------
# A.1  pack / unpack  (bit-exact)
# --------------------------------------------------------------------------
def unpack(packed: np.ndarray, bits: int) -> np.ndarray:
    """quanto::unpack -- optimum/quanto/library/unpack.py:40-54.

    plane_i = (packed >> bits*i) & (2**bits - 1); planes concatenated along dim 0.
    """
    if bits not in (2, 4):
        raise ValueError("bits must be 2 or 4")
    p = np.asarray(packed, dtype=np.uint8)
    mask = (1 << bits) - 1
    planes = [((p >> (bits * i)) & mask).astype(np.uint8) for i in range(8 // bits)]
    return np.concatenate(planes, axis=0)


def pack_weights(u: np.ndarray, bits: int) -> np.ndarray:
    """pack_weights -- optimum/quanto/tensor/packed.py:45-69.

    R = ceil(rows / (8/bits)); packed[:len] |= u[i*R:(i+1)*R] << bits*i.
    """
    u = np.asarray(u, dtype=np.uint8)
    vpi = 8 // bits
    rows = u.shape[0]
    r = (rows + vpi - 1) // vpi
    packed = np.zeros((r,) + u.shape[1:], dtype=np.uint8)
    for i in range(vpi):
        start, end = i * r, min((i + 1) * r, rows)
        if end > start:
            packed[: end - start] |= (u[start:end].astype(np.uint8) << (bits * i)).astype(np.uint8)
    return packed


def packed_unpack(packed: np.ndarray, bits: int, rows: int) -> np.ndarray:
    """PackedTensor.unpack -- optimum/quanto/tensor/packed.py:101-104 (slice to the original row count)."""
    return unpack(packed, bits)[:rows]


# --------------------------------------------------------------------------
# grouping (axis 0 only is on the hot path; -1 kept for completeness)
# --------------------------------------------------------------------------
def group(base: np.ndarray, axis: int, group_size: int) -> np.ndarray:
    """group -- optimum/quanto/tensor/grouped.py:17-30."""
    if axis == 0:
        return base.reshape(-1, group_size)
    axis_dim = base.shape[axis]
    axis_groups = base.size // axis_dim // group_size
    g = base.reshape(axis_groups, group_size, axis_dim).transpose(1, 2, 0)
    return g.reshape(group_size, axis_dim * axis_groups)


def ungroup(grouped: np.ndarray, axis: int, orig_shape) -> np.ndarray:
    """ungroup -- optimum/quanto/tensor/grouped.py:36-51."""
    if tuple(grouped.shape) == tuple(orig_shape):
        return grouped
    if axis == 0:
        return grouped.reshape(orig_shape)
    group_size = grouped.shape[0]
    axis_dim = orig_shape[axis]
    axis_groups = grouped.size // axis_dim // group_size
    u = grouped.reshape(group_size, axis_dim, axis_groups).transpose(2, 0, 1)
    return u.reshape(orig_shape)


# --------------------------------------------------------------------------
# A.2  quantize_symmetric (bit-exact)
# --------------------------------------------------------------------------
def quantize_symmetric(base_f32: np.ndarray, in_tag: str, out_tag: str, scale_f32: np.ndarray) -> np.ndarray:
    """quanto::quantize_symmetric -- optimum/quanto/library/quantize.py:51-55.

    `base_f32`/`scale_f32` hold values already representable in `in_tag`; scale is
    broadcastable to base (scalar, [N,1] for axis 0, [1,N] for axis -1).
    t = round_to_in_dtype(base / scale)   (the division result is rounded to the INPUT dtype)
    int8: rint (half-to-even), clamp [-128,127]; fp8: clamp to +-finfo.max then RNE cast (the clamp matters for
    e4m3fnuz: torch's cast maps values past 248 to NaN instead of saturating).
    Returns int8 array or fp8 bit patterns (uint8).
    """
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        t = (np.asarray(base_f32, np.float32) / np.asarray(scale_f32, np.float32)).astype(np.float32)
    t = round_to(t, in_tag)
    if out_tag == "int8":
        t = np.rint(t)  # numpy rint is round-half-even like torch.round
        t = np.where(np.isnan(t), 0, t)  # 0/0 of an all-zero row: the reference's NaN -> int8 cast yields 0 (x86, CUDA)
        return np.clip(t, -128, 127).astype(np.int8)
    mx = FP8_MAX[out_tag]
    return f32_to_fp8_bits(np.clip(t, -mx, mx), out_tag)


# --------------------------------------------------------------------------
# A.5  int4 / int2 dequantisation (bit-exact) and the linear that follows
# --------------------------------------------------------------------------
def dequantize_qbits(packed: np.ndarray, bits: int, scale_bits: np.ndarray, shift, tag: str,
                     out_features: int, in_features: int, group_size: int,
                     shift_is_int: bool = False) -> np.ndarray:
    """QBitsDequantizer.forward, axis=0 -- optimum/quanto/tensor/qbits.py:27-49.

    u = unpack(packed)[:N*K/G]  shape [N*K/G, G];
    float shift : d = rnd(scale * u) ; d = rnd(d - shift)        (two roundings, in the scale dtype)
    int   shift : d = rnd(scale * (int8(u) - int8(zp)))
    then ungroup == reshape to [N, K] (grouped.py:42-44).
    Returns the storage representation of `tag` ([N,K] bits, or float32 for f32).
    """
    rows = out_features * in_features // group_size
    u = packed_unpack(packed, bits, rows).astype(np.float32)
    s = to_f32(scale_bits, tag).reshape(rows, 1)
    if shift_is_int:
        zp = np.asarray(shift).astype(np.int8).astype(np.float32).reshape(rows, 1)
        d = round_to(s * (u - zp), tag)
    else:
        z = to_f32(shift, tag).reshape(rows, 1)
        d = round_to(s * u, tag)
        d = round_to(d - z, tag)
    return from_f32(d.reshape(out_features, in_features), tag)


def linear_from_dequantized(x_f32: np.ndarray, w_f32: np.ndarray, bias_f32=None, tag: str = "bf16"):
    """QuantizedLinearFunction.forward -- optimum/quanto/tensor/function.py:42-47.

    Returns (y_exact_f64, y_rounded_storage, tol): the exact real-number result of the reference's
    GEMM operands (+ bias) in float64; that result rounded the way the reference rounds it (matmul
    result to dtype, then `+ bias` rounded again); and the per-element rounding allowance
    (half an output ulp per rounding step) any correct fp32-accumulating implementation stays within.
    """
    mm64 = np.asarray(x_f32, np.float64) @ np.asarray(w_f32, np.float64).T
    y = round_to(mm64.astype(np.float32), tag)
    tol = 0.5 * ulp(mm64, tag)
    y64 = mm64
    if bias_f32 is not None:
        y = round_to(y + np.asarray(bias_f32, np.float32), tag)
        y64 = mm64 + np.asarray(bias_f32, np.float64)
        tol = tol + 0.5 * ulp(y64, tag)
    return y64, from_f32(y, tag), tol


# --------------------------------------------------------------------------
# A.3 / A.4  qbytes_mm
# --------------------------------------------------------------------------
def qbytes_int_mm(a_i8: np.ndarray, w_i8: np.ndarray, scales_f32: np.ndarray, tag: str) -> np.ndarray:
    """qbytes_int_mm -- optimum/quanto/library/qbytes_mm.py:36-50 (bit-exact).

    acc = int32 sum_k A[m,k]*W[n,k]; out = rnd_tag(fp32(acc) * fp32(scales[n])).
    """
    acc = np.asarray(a_i8, np.int64) @ np.asarray(w_i8, np.int64).T
    acc32 = acc.astype(np.int32).astype(np.float32)
    out = (acc32 * np.asarray(scales_f32, np.float32).reshape(1, -1)).astype(np.float32)
    return from_f32(out, tag)


def qbytes_mm_operands(a_f32: np.ndarray, w_f32: np.ndarray, scales_f32: np.ndarray, tag: str):
    """Operand preparation of the python qbytes_mm -- optimum/quanto/library/qbytes_mm.py:25-33.

    A' = rnd_tag(A) ; Ws = rnd_tag(scales * rnd_tag(W))  (scales broadcast over rows of W [N,K]).
    """
    a = round_to(a_f32, tag)
    w = round_to(w_f32, tag)
    ws = round_to(np.asarray(scales_f32, np.float32).reshape(-1, 1) * w, tag)
    return a, ws


def qbytes_mm(a_f32: np.ndarray, w_f32: np.ndarray, scales_f32: np.ndarray, tag: str):
    """Python-path qbytes_mm: returns (y_exact_f64, y_rounded_storage)."""
    a, ws = qbytes_mm_operands(a_f32, w_f32, scales_f32, tag)
    y64 = a.astype(np.float64) @ ws.astype(np.float64).T
    return y64, from_f32(y64.astype(np.float32), tag)


def qbytes_mm_fp8_native(a_bits: np.ndarray, a_tag: str, w_bits: np.ndarray, w_tag: str,
                         scales_f32: np.ndarray, tag: str):
    """Exact-math statement of the fp8 x fp8 tensor path: rnd_tag(fp32(sum a*w) * scales[n]).

    This is NOT the reference's rounding order (which rounds scales*W to the output dtype first,
    qbytes_mm.py:31-33); it is the oracle for the fp8 x fp8 tensor-core kernel, whose distance
    to the reference is bounded separately in the tests.
    """
    a = fp8_bits_to_f32(a_bits, a_tag).astype(np.float64)
    w = fp8_bits_to_f32(w_bits, w_tag).astype(np.float64)
    acc = a @ w.T
    y64 = acc * np.asarray(scales_f32, np.float64).reshape(1, -1)
    return y64, from_f32(y64.astype(np.float32), tag)


def ulp(y: np.ndarray, tag: str) -> np.ndarray:
    """Spacing of `tag` around |y| (used to state output-rounding tolerances in tests)."""
    mant = {"bf16": 7, "f16": 10, "f32": 23}[tag]
    emin = {"bf16": -126, "f16": -14, "f32": -126}[tag]
    a = np.abs(np.asarray(y, np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** emin)))
    return 2.0 ** (e - mant)


def accumulate_allowance(a_f32: np.ndarray, w_f32: np.ndarray) -> np.ndarray:
    """Slack for an fp32-accumulating GEMM evaluated in any order: 2^-22 * sqrt(K) * (|A| @ |W|^T).

    (Worst case is K * 2^-24 * |A||W|^T; the statistical growth is sqrt(K).  For K = 4096 this is
    1.5e-5 of the magnitude sum -- far inside the 1e-3 the north star allows for the accumulate.)
    """
    k = a_f32.shape[-1]
    s = np.abs(np.asarray(a_f32, np.float64)) @ np.abs(np.asarray(w_f32, np.float64)).T
    return (2.0 ** -22) * np.sqrt(k) * s


# --------------------------------------------------------------------------
# Weight freeze (SURVEY 8f rank 1/2): range search, affine / symmetric quantisation, packing.  All bit-exact.
# NB the reference's arithmetic is stated for its CPU path (true IEEE division); torch's CUDA kernels divide a
# tensor by a python scalar as `a * (1/b)`, which can differ by one ulp -- the golden vectors come from the CPU path.
# --------------------------------------------------------------------------
def max_optimizer(grouped_f32: np.ndarray, tag: str, bits: int, zeropoint: bool = False):
    """MaxOptimizer on an axis-0 grouped weight [R, G] -- optimum/quanto/tensor/optimizers/max_optimizer.py:26-37
    and AffineOptimizer.__call__ (affine_optimizer.py:52-63).

    rmin/rmax per row; scale = rnd(rnd(rmax - rmin) / (2**bits - 1)); shift = -rmin;
    zeropoint: shift = uint8(clamp(rint(rnd(shift / scale)), 0, 2**bits - 1)).
    Returns (scale storage [R,1], shift storage [R,1] or uint8 [R,1]).
    """
    b = np.asarray(grouped_f32, np.float32)
    lo = b.min(axis=1, keepdims=True)
    hi = b.max(axis=1, keepdims=True)
    levels = np.float32(2 ** bits - 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        scale = round_to(round_to(hi - lo, tag) / levels, tag)
        shift = -lo
        if zeropoint:
            zp = np.clip(np.rint(round_to(shift / scale, tag)), 0, 2 ** bits - 1)
            zp = np.where(np.isnan(zp), 0, zp)  # constant group: 0/0; the reference's NaN -> uint8 cast yields 0
            return from_f32(scale, tag), zp.astype(np.uint8)
    return from_f32(scale, tag), from_f32(shift, tag)


def quantize_affine(grouped_f32: np.ndarray, tag: str, bits: int, scale_f32: np.ndarray, shift,
                    shift_is_int: bool = False) -> np.ndarray:
    """quanto::quantize_affine on an already grouped base -- optimum/quanto/library/quantize.py:63-78.

    float shift: data = rint(rnd(rnd(base + shift) / scale));  int shift: data = rnd(rint(rnd(base / scale)) + zp);
    clamp to [0, 2**bits - 1], cast to uint8.  scale / shift broadcast against base ([R,1] for axis 0).
    """
    b = np.asarray(grouped_f32, np.float32)
    s = np.asarray(scale_f32, np.float32)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        if shift_is_int:
            zp = np.asarray(shift).astype(np.float32)
            data = round_to(np.rint(round_to(b / s, tag)) + zp, tag)
        else:
            z = np.asarray(shift, np.float32)
            data = np.rint(round_to(round_to(b + z, tag) / s, tag))
    data = np.where(np.isnan(data), 0, data)  # the reference's NaN -> uint8 cast is undefined; x86 gives 0
    return np.clip(data, 0, 2 ** bits - 1).astype(np.uint8)


def absmax_scale(base_f32: np.ndarray, tag: str, qmax: float, per_row: bool) -> np.ndarray:
    """AbsmaxOptimizer -- optimum/quanto/tensor/optimizers/absmax_optimizer.py:29-36: rnd(amax(|base|) / qmax).

    per_row: axis 0 of a 2-D base (scale [N,1]); else per-tensor (scalar).  qmax: 127 for qint8, finfo.max for float8
    (optimum/quanto/tensor/qtype.py).  Returns the storage representation of `tag`.
    """
    a = np.abs(np.asarray(base_f32, np.float32))
    top = a.reshape(a.shape[0], -1).max(axis=1, keepdims=True) if per_row else a.max()
    return from_f32(np.asarray(top / np.float32(qmax), np.float32), tag)
