"""The two `torch.ops.quanto.*` ops that keep per-tensor quantized activations quantized through attention
(the reference's ActivationQBytesTensor table, optimum/quanto/tensor/activations/qbytes_ops.py):

  quanto::qbytes_bmm      aten.bmm of two qint8 activations (qbytes_ops.py:175-186): exact int32 sum, one fp32 multiply
                          by rnd_dt(scale_a * scale_b), one rounding to the scale dtype dt
  quanto::qbytes_softmax  aten._softmax over the last dim of a quantized activation, re-quantized with the scale 1 / qmax
                          (qbytes_ops.py:208-215): codes in, codes out, one launch

Defined here rather than in library.py so that each module registers and fakes exactly the ops it defines.  As there,
only the CUDA dispatch key gets a kernel and every op has a fake implementation for torch.compile.
"""
import torch

from . import _native as N
from .library import _FLOATS, _bind_cuda, _define, _lib

__all__ = []

_define("qbytes_bmm", "(Tensor A, Tensor B, Tensor scale_a, Tensor scale_b) -> Tensor")
_define("qbytes_softmax", "(Tensor data, Tensor scale, Tensor out_scale) -> Tensor")

_CODES = (torch.int8, torch.float8_e4m3fn, torch.float8_e5m2, torch.float8_e4m3fnuz)


# ---------------------------------------------------------------------------------------------- qbytes_bmm
def _check_qbytes_bmm(a, b, scale_a, scale_b):
    if a.ndim != 3 or b.ndim != 3 or a.shape[0] != b.shape[0] or a.shape[2] != b.shape[1]:
        raise ValueError(f"qbytes_bmm expects A [B, M, K] and B [B, K, N] (got {tuple(a.shape)} and {tuple(b.shape)})")
    if a.dtype != torch.int8 or b.dtype != torch.int8:
        raise NotImplementedError(f"qbytes_bmm: int8 x int8 only (got {a.dtype} x {b.dtype})")
    if scale_a.dtype not in _FLOATS or scale_b.dtype != scale_a.dtype:
        raise ValueError(f"qbytes_bmm: scales must share one floating point dtype ({scale_a.dtype}, {scale_b.dtype})")
    if scale_a.numel() != 1 or scale_b.numel() != 1:
        raise ValueError("qbytes_bmm: activations are quantized per tensor (one scale each)")


def _batch_stride(t) -> int:
    """0 when every batch reads the same matrix (one batch, or an expanded operand), else the stride of the batch."""
    return 0 if t.shape[0] == 1 else t.stride(0)


def _b_layout(b):
    """(tensor, layout, batch stride) of B [Bt, K, N] as the kernel reads it: layout 0 = K-contiguous (element (k, n) at
    n * K + k), 1 = N-contiguous.  Any other layout is copied to a contiguous (N-contiguous) tensor first."""
    _, k, n = b.shape
    _, sk, sn = b.stride()
    bs = _batch_stride(b)
    if bs in (0, n * k):
        if (sk == 1 or k == 1) and (sn == k or n == 1):
            return b, 0, bs
        if (sn == 1 or n == 1) and (sk == n or k == 1):
            return b, 1, bs
    b = b.contiguous()
    return b, 1, _batch_stride(b)


def qbytes_bmm_cuda(a: torch.Tensor, b: torch.Tensor, scale_a: torch.Tensor, scale_b: torch.Tensor) -> torch.Tensor:
    """out[i] = rnd_dt(f32(A[i] @ B[i]) * f32(rnd_dt(scale_a * scale_b))) with an exact integer sum: bit-identical to the
    reference's fp32 bmm whenever K <= 1024 (every partial sum is then exact in fp32), deterministic above."""
    _check_qbytes_bmm(a, b, scale_a, scale_b)
    bt, m, k = a.shape
    n = b.shape[2]
    if not (a.stride(2) == 1 or k == 1) or not (a.stride(1) == k or m == 1) or _batch_stride(a) not in (0, m * k):
        a = a.contiguous()
    b, layout, b_bs = _b_layout(b)
    sa = scale_a.reshape(1).contiguous()
    sb = scale_b.reshape(1).contiguous()
    out = torch.empty((bt, m, n), dtype=scale_a.dtype, device=a.device)
    with torch.cuda.device(a.device):
        lib = N.load()
        ws_bytes = lib.qb200_qbytes_bmm_workspace_bytes(bt, n, k, b_bs, layout)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=a.device) if ws_bytes > 0 else None
        N.check(lib.qb200_qbytes_bmm(N.ptr(a), N.ptr(b), N.ptr(sa), N.ptr(sb), N.ptr(out), N.ptr(ws), ws_bytes, bt, m,
                                     n, k, _batch_stride(a), b_bs, layout, N.DTYPE_CODE[scale_a.dtype],
                                     N.stream_ptr(a.device)), "quanto::qbytes_bmm")
    return out


# ------------------------------------------------------------------------------------------ qbytes_softmax
def _check_qbytes_softmax(data, scale, out_scale):
    if data.dtype not in _CODES:
        raise NotImplementedError(f"qbytes_softmax: no sm_90a kernel for codes of dtype {data.dtype}")
    if scale.dtype not in _FLOATS or out_scale.dtype != scale.dtype:
        raise ValueError(f"qbytes_softmax: scales must share one floating point dtype ({scale.dtype}, {out_scale.dtype})")
    if scale.numel() != 1 or out_scale.numel() != 1:
        raise ValueError("qbytes_softmax: activations are quantized per tensor (one scale each)")


def qbytes_softmax_cuda(data: torch.Tensor, scale: torch.Tensor, out_scale: torch.Tensor) -> torch.Tensor:
    """quantize_symmetric(softmax(scale * data, dim=-1), data.dtype, None, out_scale) in one launch."""
    _check_qbytes_softmax(data, scale, out_scale)
    x = data.contiguous()
    out = torch.empty(x.shape, dtype=x.dtype, device=x.device)
    cols = x.shape[-1] if x.ndim > 0 else 1
    if x.numel() == 0:
        return out
    rows = x.numel() // cols
    s = scale.reshape(1).contiguous()
    qs = out_scale.reshape(1).contiguous()
    with torch.cuda.device(x.device):
        lib = N.load()
        N.check(lib.qb200_qbytes_softmax(N.ptr(x), N.ptr(s), N.ptr(qs), N.ptr(out), rows, cols, N.DTYPE_CODE[x.dtype],
                                         N.DTYPE_CODE[scale.dtype], N.stream_ptr(x.device)), "quanto::qbytes_softmax")
    return out


_bind_cuda("qbytes_bmm", qbytes_bmm_cuda)
_bind_cuda("qbytes_softmax", qbytes_softmax_cuda)


# ------------------------------------------------------------------------------------------ fake implementations
def _qbytes_bmm_fake(a, b, scale_a, scale_b):
    _check_qbytes_bmm(a, b, scale_a, scale_b)
    return a.new_empty((a.shape[0], a.shape[1], b.shape[2]), dtype=scale_a.dtype)


def _qbytes_softmax_fake(data, scale, out_scale):
    _check_qbytes_softmax(data, scale, out_scale)
    return data.new_empty(data.shape)


FAKE_IMPLS = {
    "qbytes_bmm": _qbytes_bmm_fake,
    "qbytes_softmax": _qbytes_softmax_fake,
}
for _name, _fake in FAKE_IMPLS.items():
    torch.library.register_fake("quanto::" + _name, _fake, lib=_lib)
