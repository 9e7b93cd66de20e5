"""CPU oracle of the quantized-attention ops (optimum/quanto/tensor/activations/qbytes_ops.py).  TEST INFRASTRUCTURE
ONLY; numpy, bit patterns next to dtype tags as in quanto_oracle.py, pinned to the reference by
tests/golden/qattention.npz (oracle/gen_golden_qattention.py).
"""
from __future__ import annotations

import numpy as np

from .quanto_oracle import FP8_MAX, from_f32, quantize_symmetric, round_to, to_f32  # noqa: F401 (re-exported)

QMAX = {"int8": 127.0, **FP8_MAX}
MIDPOINT_REL = 1e-5


def qbytes_bmm(a_i8: np.ndarray, b_i8: np.ndarray, sa_f32: float, sb_f32: float, tag: str) -> np.ndarray:
    """bmm of two qint8 activations -- qbytes_ops.py:175-186, with the sum in int64 (exact):
    out[b] = rnd_tag(f32(A[b] @ B[b]) * f32(rnd_tag(sa * sb))).  A [Bt, M, K], B [Bt, K, N] int8."""
    acc = np.matmul(np.asarray(a_i8, np.int64), np.asarray(b_i8, np.int64))
    s = round_to(np.float32(sa_f32) * np.float32(sb_f32), tag).astype(np.float32)
    return from_f32((acc.astype(np.float32) * s).astype(np.float32), tag)


def decode(codes: np.ndarray, q_tag: str) -> np.ndarray:
    """The payload of 8-bit codes as float32 (int8 values, or the fp8 bit patterns' values)."""
    if q_tag == "int8":
        return np.asarray(codes).view(np.int8).astype(np.float32)
    return to_f32(np.asarray(codes).view(np.uint8), q_tag)


def softmax_out_scale(q_tag: str, tag: str) -> np.ndarray:
    """torch.tensor(1 / qmax, dtype) (qbytes_ops.py:214), as the storage representation of `tag`."""
    return from_f32(np.float32(1.0 / QMAX[q_tag]), tag)


def qbytes_softmax(codes: np.ndarray, q_tag: str, scale_f32: float, tag: str):
    """_softmax of a quantized activation over the last dim -- qbytes_ops.py:208-215 -- from the float64 softmax of the
    dequantized values x = rnd_tag(scale * payload).  Returns (codes, flags): flags marks the elements whose float64
    softmax lies within 1e-5 relative of a rounding boundary of the chain (a dt rounding midpoint or a code boundary),
    where an implementation with fp32 exp / sum may land one code away."""
    x = round_to(np.float32(scale_f32) * decode(codes, q_tag), tag).astype(np.float64)
    m = np.max(x, axis=-1, keepdims=True)
    e = np.exp(x - m)
    p = e / np.sum(e, axis=-1, keepdims=True)
    os_f32 = to_f32(softmax_out_scale(q_tag, tag), tag)

    def quantize(v):
        return quantize_symmetric(round_to(v.astype(np.float32), tag), tag, q_tag, os_f32)

    out = quantize(p)
    lo, hi = quantize(p * (1 - MIDPOINT_REL)), quantize(p * (1 + MIDPOINT_REL))
    flags = (lo != out) | (hi != out)
    return out, flags


def code_distance(a: np.ndarray, b: np.ndarray, q_tag: str) -> np.ndarray:
    """|a - b| in codes: int8 values, or positions on the fp8 number line (sign-magnitude -> ordered integers)."""
    if q_tag == "int8":
        return np.abs(np.asarray(a).view(np.int8).astype(np.int32) - np.asarray(b).view(np.int8).astype(np.int32))

    def ordered(c):
        c = np.asarray(c).view(np.uint8).astype(np.int32)
        return np.where(c & 0x80, -(c & 0x7F), c & 0x7F)

    return np.abs(ordered(a) - ordered(b))


def layout_result(shape, stride, op: str, *args):
    """(shape, strides) of a layout op applied to a tensor of `shape` / `stride` (elements): what the table hands back
    as the outer shape and strides of the quantized result."""
    a = np.lib.stride_tricks.as_strided(np.zeros(1, np.int8), shape=shape, strides=stride, writeable=False)
    if op == "transpose":
        r = np.swapaxes(a, *args)
    elif op == "permute":
        r = np.transpose(a, args[0])
    elif op == "select":
        index = [slice(None)] * a.ndim
        index[args[0]] = args[1]
        r = a[tuple(index)]
    elif op == "expand":
        r = np.broadcast_to(a, args[0])
    else:
        raise ValueError(op)
    return tuple(r.shape), tuple(r.strides)  # int8: byte strides are element strides
