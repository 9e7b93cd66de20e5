"""`torch.ops.quanto.*` registry backed by the sm_90a kernels (C-ABI in include/quanto_b200.h).

Keeps the reference's op names and schemas so that QTensor code written against quanto keeps working:
  quanto::unpack             optimum/quanto/library/unpack.py:18
  quanto::qbytes_mm          optimum/quanto/library/qbytes_mm.py:22
  quanto::quantize_symmetric optimum/quanto/library/quantize.py:22-24
  quanto::quantize_affine    optimum/quanto/library/quantize.py:58-61   (CUDA kernel; ATen composition elsewhere, as upstream)
adds the two fused ops that take the place of the retired AWQ / Marlin / TinyGemm bindings
(optimum/quanto/library/extensions/cuda/__init__.py:82-202):
  quanto::qbits_mm           fused packed-int4 linear (the `udqmm` role)
  quanto::dequantize_qbits   unpack + scale + shift + ungroup in one launch
  quanto::qbytes_linear      qbytes_mm with the bias of the 8-bit linear fused into the epilogue
  quanto::qbytes_linear_quantized  ... and the per-tensor output quantisation too (quantized activations in and out)
the input gradients of the two quantized linears (the backward's gO @ W, reading the quantized weights):
  quanto::qbits_grad_input   packed int4 weights
  quanto::qbytes_grad_input  int8 / float8 weights
and the weight-freeze / calibration ops of the step before the path (SURVEY.md 8f):
  quanto::pack                    pack_weights (optimum/quanto/tensor/packed.py:24-69) as one launch
  quanto::quantize_qbits_max      MaxOptimizer + quantize_affine + pack_weights in one launch (axis 0)
  quanto::quantize_qbytes_absmax  AbsmaxOptimizer + quantize_symmetric in one launch (axis 0)
  quanto::quantize_qbits_hqq      HqqOptimizer + quantize_affine + pack_weights in two launches (axis 0)
  quanto::hqq_shrink              shrink_lp_op of HqqOptimizer (optimum/quanto/tensor/optimizers/hqq_optimizer.py:28-34)
  quanto::absmax                  per-tensor max|x| (optimum/quanto/calibrate.py:37-61)

Only the CUDA dispatch key gets a kernel.  There is deliberately no CPU implementation of the hot-path ops: calling
them with CPU tensors raises NotImplementedError from the dispatcher, and a missing native library raises at first use.
(`quanto::quantize_affine` -- weight preparation, not the forward path -- keeps upstream's python composition for CPU
tensors, as optimum/quanto/library/quantize.py:63-78 does, so that a module can be frozen before it is moved.)
If the reference package was imported first, its definitions are reused and only the CUDA kernels are (re)bound.
Every op also has a fake implementation (end of this file) so that torch.compile / AOTAutograd can trace it.
"""
from typing import Optional

import torch

from . import _native as N
from .tensor.core import dtype_info
from .tensor.grouped import group

__all__ = []

_lib = torch.library.Library("quanto", "FRAGMENT")


def _defined(name: str) -> bool:
    try:
        getattr(torch.ops.quanto, name)
        return True
    except (AttributeError, RuntimeError):
        return False


def _define(name: str, schema: str):
    if not _defined(name):
        _lib.define(name + schema)


_define("unpack", "(Tensor self, int bits) -> Tensor")
_define("qbytes_mm", "(Tensor A, Tensor B, Tensor scales) -> Tensor")
_define("quantize_symmetric", "(Tensor base, ScalarType dtype, int? axis, Tensor scale) -> Tensor")
_define("quantize_affine", "(Tensor base, int bits, int axis, int? group_size, Tensor scale, Tensor shift) -> Tensor")
_define("qbits_mm", "(Tensor A, Tensor packed, Tensor scale, Tensor shift, Tensor? bias, int out_features, "
                    "int group_size, int bits=4) -> Tensor")
_define("dequantize_qbits", "(Tensor packed, Tensor scale, Tensor shift, int out_features, int in_features, "
                            "int group_size, int bits) -> Tensor")
_define("qbytes_linear", "(Tensor A, Tensor B, Tensor scales, Tensor? bias) -> Tensor")
_define("qbytes_linear_quantized", "(Tensor A, Tensor B, Tensor scales, Tensor? bias, Tensor out_scale, "
                                   "ScalarType out_dtype) -> Tensor")
_define("pack", "(Tensor self, int bits) -> Tensor")
_define("quantize_qbits_max", "(Tensor base, int bits, int group_size, bool zeropoint) -> (Tensor, Tensor, Tensor)")
_define("quantize_qbytes_absmax", "(Tensor base, ScalarType dtype) -> (Tensor, Tensor)")
_define("absmax", "(Tensor base) -> Tensor")
_define("quantize_qbits_hqq", "(Tensor base, int bits, int group_size, bool zeropoint, float lp_norm, float beta, "
                              "float kappa, int iters) -> (Tensor, Tensor, Tensor, Tensor)")
_define("hqq_shrink", "(Tensor x, float beta, float lp_norm) -> Tensor")
_define("qbits_grad_input", "(Tensor grad_output, Tensor packed, Tensor scale, Tensor shift, int out_features, "
                            "int group_size, int bits) -> Tensor")
_define("qbytes_grad_input", "(Tensor grad_output, Tensor B, Tensor scales) -> Tensor")


def _require_contiguous(t: torch.Tensor, what: str) -> torch.Tensor:
    return t if t.is_contiguous() else t.contiguous()


# --------------------------------------------------------------------------------------------- unpack
def _unpack_shape(packed, bits: int):
    if packed.dtype != torch.uint8:
        raise RuntimeError("Unsupported argument dtype: expected torch.uint8")  # mirrors unpack.cu:86-88
    if bits not in (2, 4):
        raise ValueError("Can only unpack 2-bit or 4-bit values")
    return (packed.shape[0] * (8 // bits),) + tuple(packed.shape[1:])


def unpack_cuda(packed: torch.Tensor, bits: int) -> torch.Tensor:
    shape = _unpack_shape(packed, bits)
    packed = _require_contiguous(packed, "packed")
    out = torch.empty(shape, dtype=torch.uint8, device=packed.device)
    with torch.cuda.device(packed.device):
        lib = N.load()
        N.check(lib.qb200_unpack(N.ptr(packed), N.ptr(out), packed.numel(), bits, N.stream_ptr(packed.device)),
                "quanto::unpack")
    return out


# --------------------------------------------------------------------------------- quantize_symmetric
def _check_symmetric_args(base, axis, scale):
    """Same validation and messages as optimum/quanto/library/quantize.py:32-50."""
    if axis is None:
        if scale.ndim > 0:
            raise ValueError("Scale must be a scalar when quantizing per-tensor")
        return None
    if base.ndim == 1:
        raise ValueError("1D Tensors cannot be quantized per-axis")
    if axis == base.ndim - 1:
        axis = -1
    if axis not in (0, -1):
        raise ValueError("Quantization is only supported along the first or last axis.")
    if base.shape[axis] == 1:
        raise ValueError(f"Cannot quantize Tensor of shape {base.shape} along axis {axis} of size 1")
    if torch.squeeze(scale).ndim > 1:
        raise ValueError("Quantizing along multiple axis is not supported")
    if scale.ndim != base.ndim:
        raise ValueError(
            "When quantizing per-axis, the scale must be broadcastable to the base (Tip: try to add missing dims of length zero)."
        )
    return axis


def _quantize_symmetric_plan(base, dtype, axis, scale):
    """Argument checks of quanto::quantize_symmetric -> (outer, inner, mode) of the kernel's [outer, inner] view."""
    axis = _check_symmetric_args(base, axis, scale)
    if base.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise ValueError(f"quantize_symmetric: unsupported base dtype {base.dtype}")
    if dtype not in (torch.int8, torch.float8_e4m3fn, torch.float8_e5m2, torch.float8_e4m3fnuz):
        raise NotImplementedError(f"quantize_symmetric: no sm_90a kernel for target dtype {dtype}")
    if axis is None:
        outer, inner, mode = 1, base.numel(), 0
        if scale.numel() != 1:
            raise ValueError("Scale must be a scalar when quantizing per-tensor")
    elif axis == 0:
        outer, mode = base.shape[0], 1
        inner = base.numel() // max(outer, 1)
        if scale.numel() != outer:
            raise ValueError("scale does not match the quantization axis")
    else:
        inner, mode = base.shape[-1], 2
        outer = base.numel() // max(inner, 1)
        if scale.numel() != inner:
            raise ValueError("scale does not match the quantization axis")
    return outer, inner, mode


def quantize_symmetric_cuda(base: torch.Tensor, dtype: torch.dtype, axis: Optional[int], scale: torch.Tensor):
    outer, inner, mode = _quantize_symmetric_plan(base, dtype, axis, scale)
    base = _require_contiguous(base, "base")
    scale = scale.to(base.dtype).reshape(-1).contiguous()
    out = torch.empty(base.shape, dtype=dtype, device=base.device)
    with torch.cuda.device(base.device):
        lib = N.load()
        N.check(lib.qb200_quantize_symmetric(N.ptr(base), N.ptr(scale), N.ptr(out), outer, inner, mode,
                                             N.DTYPE_CODE[base.dtype], N.DTYPE_CODE[dtype],
                                             N.stream_ptr(base.device)), "quanto::quantize_symmetric")
    return out


# ----------------------------------------------------------------------------------- quantize_affine
_FLOATS = (torch.float32, torch.float16, torch.bfloat16)


def _quantize_affine_aten(grouped, bits: int, scale, shift):
    """ATen composition on the grouped base, same arithmetic as optimum/quanto/library/quantize.py:71-78."""
    if shift.dtype.is_floating_point:
        data = torch.round((grouped + shift) / scale)
    else:
        data = torch.round(grouped / scale) + shift
    return torch.clamp(data, min=0, max=2**bits - 1).to(torch.uint8)


def quantize_affine_any(base, bits: int, axis: int, group_size: Optional[int], scale, shift):
    """ATen composition (any device), as upstream (optimum/quanto/library/quantize.py:63-78)."""
    if axis not in (0, -1):
        raise ValueError("axis parameter must be 0 (first axis) or -1 (last axis)")
    if group_size is not None:
        base = group(base, axis=axis, group_size=group_size)
    return _quantize_affine_aten(base, bits, scale, shift)


def _affine_mode(grouped, scale, shift):
    """0 / 1 / 2 = one, per-row, per-column scale+shift of a 2-D grouped base; None = a broadcast the kernel lacks."""
    if grouped.ndim != 2 or scale.shape != shift.shape or grouped.dtype not in _FLOATS or scale.dtype != grouped.dtype:
        return None
    if not (shift.dtype == grouped.dtype or shift.dtype in (torch.uint8, torch.int8)):
        return None
    rows, cols = grouped.shape
    if scale.numel() == 1:
        return 0
    if tuple(scale.shape) == (rows, 1):
        return 1
    if tuple(scale.shape) == (1, cols):
        return 2
    return None


def _quantize_affine_plan(base, bits: int, axis: int, group_size: Optional[int], scale, shift):
    """(grouped base, kernel mode); mode None = the ATen composition runs instead of the kernel."""
    if axis not in (0, -1):
        raise ValueError("axis parameter must be 0 (first axis) or -1 (last axis)")
    grouped = base if group_size is None else group(base, axis=axis, group_size=group_size)
    mode = _affine_mode(grouped, scale, shift)
    return grouped, (mode if 1 <= bits <= 8 else None)


def quantize_affine_cuda(base, bits: int, axis: int, group_size: Optional[int], scale, shift):
    """One launch instead of the 4-5 ATen kernels of the reference composition; bit-exact with its CPU arithmetic."""
    grouped, mode = _quantize_affine_plan(base, bits, axis, group_size, scale, shift)
    if mode is None:
        return _quantize_affine_aten(grouped, bits, scale, shift)
    grouped = _require_contiguous(grouped, "base")
    scale_f = scale.reshape(-1).contiguous()
    shift_f = shift.reshape(-1).contiguous()
    # zero-points are added by VALUE (library/quantize.py:74-76): 1 = uint8 payload, 2 = int8 payload (may be negative)
    shift_is_int = 0 if shift_f.dtype.is_floating_point else (2 if shift_f.dtype == torch.int8 else 1)
    if shift_f.dtype == torch.int8:
        shift_f = shift_f.view(torch.uint8)
    out = torch.empty(grouped.shape, dtype=torch.uint8, device=grouped.device)
    with torch.cuda.device(grouped.device):
        lib = N.load()
        N.check(lib.qb200_quantize_affine(N.ptr(grouped), N.ptr(scale_f), N.ptr(shift_f), N.ptr(out), grouped.shape[0],
                                          grouped.shape[1], mode, bits, N.DTYPE_CODE[grouped.dtype], shift_is_int,
                                          N.stream_ptr(grouped.device)), "quanto::quantize_affine")
    return out


# ------------------------------------------------------------------ pack / fused freeze / absmax (SURVEY 8f)
def _pack_shape(values, bits: int):
    if values.dtype not in (torch.uint8, torch.int8):
        raise RuntimeError("Unsupported argument dtype: expected torch.uint8")
    if bits not in (2, 4):
        raise ValueError("bits must be 2 or 4")
    return (-(-values.shape[0] // (8 // bits)),) + tuple(values.shape[1:])


def _freeze_qbits_shapes(what: str, base, bits: int, group_size: int, zeropoint: bool):
    """Checks of the fused qint4 / qint2 freeze ops -> (packed shape, scale / shift shape, shift dtype)."""
    if base.ndim != 2:
        raise ValueError(f"{what} expects a 2-D weight [out_features, in_features]")
    if base.dtype not in _FLOATS:
        raise ValueError(f"{what}: unsupported dtype {base.dtype}")
    if bits not in (2, 4):
        raise ValueError("bits must be 2 or 4")
    n, k = base.shape
    if group_size <= 0 or k % group_size != 0:
        raise ValueError(f"Group size ({group_size}) must be a divisor of ({k})")
    rows = n * k // group_size
    return (-(-rows // (8 // bits)), group_size), (rows, 1), (torch.uint8 if zeropoint else base.dtype)


def pack_cuda(values: torch.Tensor, bits: int) -> torch.Tensor:
    """pack_weights (optimum/quanto/tensor/packed.py:24-69) as one launch; the inverse of quanto::unpack + [:rows]."""
    shape = _pack_shape(values, bits)
    values = _require_contiguous(values, "values")
    if values.dtype == torch.int8:
        values = values.view(torch.uint8)
    rows = values.shape[0]
    cols = values.numel() // rows if rows else 0
    out = torch.empty(shape, dtype=torch.uint8, device=values.device)
    with torch.cuda.device(values.device):
        lib = N.load()
        N.check(lib.qb200_pack(N.ptr(values), N.ptr(out), rows, cols, bits, N.stream_ptr(values.device)),
                "quanto::pack")
    return out


def quantize_qbits_max_cuda(base: torch.Tensor, bits: int, group_size: int, zeropoint: bool):
    """MaxOptimizer + quantize_affine + pack_weights for an axis-0 weight [N, K] in one launch.

    Returns (packed [ceil(R / (8/bits)), G] uint8, scale [R, 1], shift [R, 1] (base dtype, or uint8 zero-points)),
    R = N*K/G: exactly the inner tensors of the reference's `WeightQBitsTensor` for `MaxOptimizer()` scales
    (optimum/quanto/tensor/optimizers/max_optimizer.py:26-37, affine_optimizer.py:52-63, library/quantize.py:63-78,
    tensor/packed.py:45-69).  Raises UnsupportedConfiguration for group sizes the kernel does not take.
    """
    packed_shape, coef_shape, shift_dtype = _freeze_qbits_shapes("quantize_qbits_max", base, bits, group_size, zeropoint)
    n, k = base.shape
    base = _require_contiguous(base, "base")
    packed = torch.empty(packed_shape, dtype=torch.uint8, device=base.device)
    scale = torch.empty(coef_shape, dtype=base.dtype, device=base.device)
    shift = torch.empty(coef_shape, dtype=shift_dtype, device=base.device)
    with torch.cuda.device(base.device):
        lib = N.load()
        N.check(lib.qb200_quantize_qbits_max(N.ptr(base), N.ptr(packed), N.ptr(scale), N.ptr(shift), n, k, group_size,
                                             bits, N.DTYPE_CODE[base.dtype], 1 if zeropoint else 0,
                                             N.stream_ptr(base.device)), "quanto::quantize_qbits_max")
    return packed, scale, shift


def quantize_qbits_hqq_cuda(base: torch.Tensor, bits: int, group_size: int, zeropoint: bool, lp_norm: float,
                            beta: float, kappa: float, iters: int):
    """HqqOptimizer + quantize_affine + pack_weights for an axis-0 weight [N, K] in two launches, no host sync.

    Returns (packed, scale, shift) as quanto::quantize_qbits_max does, for the scale and shift that
    `HqqOptimizer(lp_norm, beta, kappa, iters)(base, qtype, axis=0, group_size, zeropoint)` returns
    (optimum/quanto/tensor/optimizers/hqq_optimizer.py:60-87), and `errors` (float32 [iters + 2]): the dt-rounded mean
    errors of the all-accepted trajectory (start error, then one per iteration), then the accepted count.  Raises
    UnsupportedConfiguration for what the kernel does not take (float32, group > 256, iters > 64, ...).
    """
    packed_shape, coef_shape, shift_dtype = _freeze_qbits_shapes("quantize_qbits_hqq", base, bits, group_size, zeropoint)
    n, k = base.shape
    base = _require_contiguous(base, "base")
    packed = torch.empty(packed_shape, dtype=torch.uint8, device=base.device)
    scale = torch.empty(coef_shape, dtype=base.dtype, device=base.device)
    shift = torch.empty(coef_shape, dtype=shift_dtype, device=base.device)
    errors = torch.empty(max(iters, 0) + 2, dtype=torch.float32, device=base.device)
    with torch.cuda.device(base.device):
        lib = N.load()
        ws_bytes = lib.qb200_quantize_qbits_hqq_workspace_bytes(n, k, group_size, iters)
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=base.device)
        N.check(lib.qb200_quantize_qbits_hqq(N.ptr(base), N.ptr(packed), N.ptr(scale), N.ptr(shift), N.ptr(errors),
                                             N.ptr(ws), n, k, group_size, bits, N.DTYPE_CODE[base.dtype],
                                             1 if zeropoint else 0, lp_norm, beta, kappa, iters,
                                             N.stream_ptr(base.device)), "quanto::quantize_qbits_hqq")
    return packed, scale, shift, errors


def _check_float(what: str, x):
    if x.dtype not in _FLOATS:
        raise ValueError(f"{what}: unsupported dtype {x.dtype}")


def hqq_shrink_cuda(x: torch.Tensor, beta: float, lp_norm: float) -> torch.Tensor:
    """shrink_lp_op(x, beta, lp_norm) (optimum/quanto/tensor/optimizers/hqq_optimizer.py:28-34) with the device
    arithmetic quanto::quantize_qbits_hqq uses; bf16 / fp16."""
    _check_float("hqq_shrink", x)
    x = _require_contiguous(x, "x")
    out = torch.empty_like(x)
    with torch.cuda.device(x.device):
        lib = N.load()
        N.check(lib.qb200_hqq_shrink(N.ptr(x), N.ptr(out), x.numel(), beta, lp_norm, N.DTYPE_CODE[x.dtype],
                                     N.stream_ptr(x.device)), "quanto::hqq_shrink")
    return out


def _check_qbytes_absmax(base, dtype):
    if base.ndim != 2:
        raise ValueError("quantize_qbytes_absmax expects a 2-D weight [out_features, in_features]")
    _check_float("quantize_qbytes_absmax", base)
    if dtype not in (torch.int8, torch.float8_e4m3fn, torch.float8_e5m2):
        raise NotImplementedError(f"quantize_qbytes_absmax: no sm_90a kernel for target dtype {dtype}")


def quantize_qbytes_absmax_cuda(base: torch.Tensor, dtype: torch.dtype):
    """AbsmaxOptimizer + quantize_symmetric for an axis-0 weight [N, K] in one launch: (data [N, K], scale [N, 1])."""
    _check_qbytes_absmax(base, dtype)
    base = _require_contiguous(base, "base")
    n, k = base.shape
    data = torch.empty((n, k), dtype=dtype, device=base.device)
    scale = torch.empty((n, 1), dtype=base.dtype, device=base.device)
    with torch.cuda.device(base.device):
        lib = N.load()
        N.check(lib.qb200_quantize_qbytes_absmax(N.ptr(base), N.ptr(data), N.ptr(scale), n, k,
                                                 N.DTYPE_CODE[base.dtype], N.DTYPE_CODE[dtype],
                                                 N.stream_ptr(base.device)), "quanto::quantize_qbytes_absmax")
    return data, scale


def absmax_cuda(base: torch.Tensor) -> torch.Tensor:
    """max |base| over the whole tensor, as a 0-dim tensor of base.dtype (one launch + an 8-byte memset)."""
    _check_float("absmax", base)
    base = _require_contiguous(base, "base")
    out = torch.empty((), dtype=base.dtype, device=base.device)
    scratch = torch.empty(2, dtype=torch.int32, device=base.device)
    with torch.cuda.device(base.device):
        lib = N.load()
        N.check(lib.qb200_absmax(N.ptr(base), N.ptr(out), N.ptr(scratch), base.numel(), N.DTYPE_CODE[base.dtype],
                                 N.stream_ptr(base.device)), "quanto::absmax")
    return out


# ----------------------------------------------------------------------------------------- qbytes_mm
def _check_qbytes_mm(activations, weights, output_scales):
    if activations.ndim < 1 or weights.ndim != 2:
        raise ValueError("qbytes_mm expects activations [..., K] and weights [N, K]")
    n, k = weights.shape
    if activations.shape[-1] != k:
        raise ValueError(f"qbytes_mm: in_features mismatch ({activations.shape[-1]} vs {k})")
    if weights.dtype not in (torch.int8, torch.float8_e4m3fn, torch.float8_e5m2, torch.float8_e4m3fnuz):
        raise NotImplementedError(f"qbytes_mm: no sm_90a kernel for weights of dtype {weights.dtype}")
    if activations.dtype not in N.DTYPE_CODE or activations.dtype == torch.uint8:
        raise NotImplementedError(f"qbytes_mm: unsupported activations dtype {activations.dtype}")
    if output_scales.dtype not in (torch.float32, torch.float16, torch.bfloat16):
        raise ValueError("qbytes_mm: scales must be floating point")
    if output_scales.numel() not in (1, n):
        raise ValueError("qbytes_mm: scales must have one value per output feature")


def qbytes_mm_cuda(activations: torch.Tensor, weights: torch.Tensor, output_scales: torch.Tensor,
                   bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    _check_qbytes_mm(activations, weights, output_scales)
    n, k = weights.shape
    out_dtype = output_scales.dtype
    a2 = _require_contiguous(activations.reshape(-1, k), "A")
    w = _require_contiguous(weights, "B")
    if output_scales.numel() == 1:
        scales = output_scales.reshape(1).expand(n).contiguous()
    else:
        scales = output_scales.reshape(-1).contiguous()
    m = a2.shape[0]
    out = torch.empty((m, n), dtype=out_dtype, device=a2.device)
    with torch.cuda.device(a2.device):
        lib = N.load()
        N.check(lib.qb200_qbytes_mm(N.ptr(a2), N.ptr(w), N.ptr(scales), N.ptr(bias), N.ptr(out), m, n, k,
                                    N.DTYPE_CODE[a2.dtype], N.DTYPE_CODE[w.dtype], N.DTYPE_CODE[out_dtype],
                                    N.stream_ptr(a2.device)), "quanto::qbytes_mm")
    return out.reshape(activations.shape[:-1] + (n,))


def _qbytes_mm_op(activations, weights, output_scales):
    return qbytes_mm_cuda(activations, weights, output_scales)


def _bias_in_epilogue(weights, output_scales, bias) -> bool:
    """False: a bias broadcast the epilogue does not do, added after the GEMM instead."""
    return bias.dtype == output_scales.dtype and bias.numel() == weights.shape[0]


def _qbytes_linear_op(activations, weights, output_scales, bias):
    """`qbytes_mm(...) + bias` of WeightQBytesLinearFunction (optimum/quanto/tensor/weights/qbytes.py:68-82) as ONE launch:
    the bias is added in the GEMM epilogue after the output was rounded to the scales' dtype (same two roundings)."""
    if bias is not None:
        if not _bias_in_epilogue(weights, output_scales, bias):
            return qbytes_mm_cuda(activations, weights, output_scales) + bias
        bias = bias.reshape(-1).contiguous()
    return qbytes_mm_cuda(activations, weights, output_scales, bias)


def _qbytes_linear_quantized_fusable(activations, weights, output_scales, bias, out_scale, out_dtype) -> bool:
    """Whether the one-launch kernel is tried; otherwise (or when it declines) the composition of native ops runs."""
    n, k = weights.shape
    scale_dtype = output_scales.dtype
    return (
        out_dtype in (torch.int8, torch.float8_e4m3fn, torch.float8_e5m2)
        and activations.dtype in (torch.int8, torch.float8_e4m3fn, torch.float8_e5m2)
        and scale_dtype in _FLOATS and out_scale.numel() == 1 and out_scale.dtype == scale_dtype
        and (bias is None or (bias.dtype == scale_dtype and bias.numel() == n))
        and activations.shape[-1] == k and output_scales.numel() == n
    )


def qbytes_linear_quantized_cuda(activations, weights, output_scales, bias, out_scale, out_dtype):
    """8-bit linear + bias + per-tensor output quantisation in ONE launch (quantized activations in AND out):
    `quantize_symmetric(qbytes_mm(A, B, scales) + bias, out_dtype, None, out_scale)`, bit for bit.  Falls back to exactly
    that composition of native kernels for problems the tensor-core kernels do not take."""
    n, k = weights.shape
    scale_dtype = output_scales.dtype
    if _qbytes_linear_quantized_fusable(activations, weights, output_scales, bias, out_scale, out_dtype):
        a2 = _require_contiguous(activations.reshape(-1, k), "A")
        w = _require_contiguous(weights, "B")
        scales = output_scales.reshape(-1).contiguous()
        bias_f = None if bias is None else bias.reshape(-1).contiguous()
        qs = out_scale.reshape(1).contiguous()
        m = a2.shape[0]
        out = torch.empty((m, n), dtype=out_dtype, device=a2.device)
        with torch.cuda.device(a2.device):
            lib = N.load()
            try:
                N.check(lib.qb200_qbytes_mm_quantized(N.ptr(a2), N.ptr(w), N.ptr(scales), N.ptr(bias_f), N.ptr(out),
                                                      N.ptr(qs), m, n, k, N.DTYPE_CODE[a2.dtype], N.DTYPE_CODE[w.dtype],
                                                      N.DTYPE_CODE[scale_dtype], N.DTYPE_CODE[out_dtype],
                                                      N.stream_ptr(a2.device)), "quanto::qbytes_linear_quantized")
                return out.reshape(activations.shape[:-1] + (n,))
            except N.UnsupportedConfiguration:
                pass
    y = _qbytes_linear_op(activations, weights, output_scales, bias)
    return quantize_symmetric_cuda(y, out_dtype, None, out_scale.reshape(()))


# -------------------------------------------------------------------------- dequantize_qbits / qbits_mm
def _check_dequantize_qbits(shift):
    if not shift.dtype.is_floating_point and shift.dtype not in (torch.uint8, torch.int8):
        raise ValueError("integer shifts must be uint8 / int8 zero-points")


def dequantize_qbits_cuda(packed, scale, shift, out_features: int, in_features: int, group_size: int, bits: int):
    _check_dequantize_qbits(shift)
    packed = _require_contiguous(packed, "packed")
    scale_f = _require_contiguous(scale.reshape(-1), "scale")
    shift_f = _require_contiguous(shift.reshape(-1), "shift")
    shift_is_int = 0 if shift_f.dtype.is_floating_point else 1
    out = torch.empty((out_features, in_features), dtype=scale.dtype, device=packed.device)
    with torch.cuda.device(packed.device):
        lib = N.load()
        N.check(lib.qb200_dequantize_qbits(N.ptr(packed), N.ptr(scale_f), N.ptr(shift_f), N.ptr(out), out_features,
                                           in_features, group_size, bits, N.DTYPE_CODE[scale.dtype], shift_is_int,
                                           N.stream_ptr(packed.device)), "quanto::dequantize_qbits")
    return out


def _check_qbits_mm(activations, packed, scale, shift, bias, out_features: int, group_size: int, bits: int):
    k = activations.shape[-1]
    if packed.dtype != torch.uint8:
        raise ValueError("qbits_mm: packed weights must be uint8")
    if activations.dtype not in _FLOATS:
        raise ValueError(f"qbits_mm: unsupported activations dtype {activations.dtype}")
    if scale.dtype != activations.dtype:
        raise ValueError(f"qbits_mm: scale dtype {scale.dtype} does not match the activations ({activations.dtype})")
    if shift.dtype.is_floating_point:
        if shift.dtype != activations.dtype:
            raise ValueError(f"qbits_mm: float shift of dtype {shift.dtype} does not match the activations")
    elif shift.dtype not in (torch.uint8, torch.int8):
        raise ValueError("qbits_mm: integer shifts must be uint8 / int8 zero-points")
    if bits not in (2, 4):
        raise ValueError("qbits_mm: bits must be 2 or 4")
    if group_size <= 0 or k % group_size != 0:
        raise ValueError(f"qbits_mm: group size {group_size} does not divide in_features {k}")
    rows = out_features * (k // group_size)
    if scale.numel() != rows or shift.numel() != rows:
        raise ValueError("qbits_mm: scale / shift must hold one value per (out_feature, group)")
    if packed.numel() != -(-rows // (8 // bits)) * group_size:
        raise ValueError("qbits_mm: packed tensor does not match out_features x in_features")
    if bias is not None and bias.numel() != out_features:
        raise ValueError("qbits_mm: bias must have one value per output feature")


def qbits_mm_cuda(activations, packed, scale, shift, bias, out_features: int, group_size: int, bits: int = 4):
    """Fused packed-int4 / int2 linear (the `udqmm` role): ONE native launch for every valid axis-0 weight.  The shapes the
    tensor-core kernels do not take run on the library's own CUDA-core kernel -- there is no eager / cuBLAS fallback."""
    _check_qbits_mm(activations, packed, scale, shift, bias, out_features, group_size, bits)
    k = activations.shape[-1]
    a2 = _require_contiguous(activations.reshape(-1, k), "A")
    packed = _require_contiguous(packed, "packed")
    scale_f = _require_contiguous(scale.reshape(-1), "scale")
    shift_f = _require_contiguous(shift.reshape(-1), "shift")
    shift_is_int = 0 if shift_f.dtype.is_floating_point else 1
    if shift_f.dtype == torch.int8:
        shift_f = shift_f.view(torch.uint8)
    if bias is not None:
        bias = _require_contiguous(bias.to(a2.dtype).reshape(-1), "bias")
    m = a2.shape[0]
    out = torch.empty((m, out_features), dtype=a2.dtype, device=a2.device)
    with torch.cuda.device(a2.device):
        lib = N.load()
        stream = N.stream_ptr(a2.device)
        ws = N.workspace(a2.device, stream, lib.qb200_qbits_mm_workspace_bytes(m, out_features, k))
        N.check(lib.qb200_qbits_mm(N.ptr(a2), N.ptr(packed), N.ptr(scale_f), N.ptr(shift_f), N.ptr(bias),
                                   N.ptr(out), m, out_features, k, group_size, bits, N.DTYPE_CODE[a2.dtype],
                                   shift_is_int, N.ptr(ws), 0 if ws is None else ws.numel(), stream),
                "quanto::qbits_mm")
    return out.reshape(activations.shape[:-1] + (out_features,))


# ------------------------------------------------------------------------- input gradients of the linears
def _check_grad_output_2d(grad_output, out_features: int, what: str):
    if grad_output.ndim != 2 or grad_output.shape[1] != out_features:
        raise ValueError(f"{what}: grad_output must be [M, {out_features}] (got {tuple(grad_output.shape)})")


def _check_qbits_grad_input(grad_output, packed, scale, shift, out_features: int, group_size: int, bits: int) -> int:
    """-> in_features K of the [M, K] input gradient."""
    if packed.dtype != torch.uint8:
        raise ValueError("qbits_grad_input: packed weights must be uint8")
    if bits not in (2, 4):
        raise ValueError("qbits_grad_input: bits must be 2 or 4")
    _check_grad_output_2d(grad_output, out_features, "qbits_grad_input")
    if grad_output.dtype != scale.dtype:
        raise ValueError(f"qbits_grad_input: grad_output dtype {grad_output.dtype} does not match the scale ({scale.dtype})")
    if shift.dtype.is_floating_point:
        if shift.dtype != scale.dtype:
            raise ValueError(f"qbits_grad_input: float shift of dtype {shift.dtype} does not match the scale")
    elif shift.dtype not in (torch.uint8, torch.int8):
        raise ValueError("qbits_grad_input: integer shifts must be uint8 / int8 zero-points")
    if group_size <= 0 or scale.numel() != shift.numel() or (scale.numel() * group_size) % out_features != 0:
        raise ValueError("qbits_grad_input: scale / shift must hold one value per (out_feature, group)")
    k = scale.numel() * group_size // out_features
    if k % group_size != 0:
        raise ValueError(f"qbits_grad_input: group size {group_size} does not divide in_features {k}")
    if packed.numel() != -(-scale.numel() // (8 // bits)) * group_size:
        raise ValueError("qbits_grad_input: packed tensor does not match out_features x in_features")
    return k


def qbits_grad_input_cuda(grad_output, packed, scale, shift, out_features: int, group_size: int, bits: int):
    """dX = gO @ dequant(W) for a canonical axis-0 packed weight: ONE native launch that reads the packed bytes.

    Shapes the kernel declines (2-bit, fp32, N % 16 != 0, K % 16 != 0, other group sizes, unaligned buffers) run the
    composition the reference's backward performs: dequantize (quanto::dequantize_qbits, bit-exact), then matmul."""
    k = _check_qbits_grad_input(grad_output, packed, scale, shift, out_features, group_size, bits)
    gO = _require_contiguous(grad_output, "grad_output")
    m = gO.shape[0]
    packed_c = _require_contiguous(packed, "packed")
    scale_f = _require_contiguous(scale.reshape(-1), "scale")
    shift_f = _require_contiguous(shift.reshape(-1), "shift")
    shift_is_int = 0 if shift_f.dtype.is_floating_point else 1
    if shift_f.dtype == torch.int8:
        shift_f = shift_f.view(torch.uint8)
    if bits == 4:
        out = torch.empty((m, k), dtype=gO.dtype, device=gO.device)
        with torch.cuda.device(gO.device):
            lib = N.load()
            try:
                N.check(lib.qb200_qbits_mm_grad_input(N.ptr(gO), N.ptr(packed_c), N.ptr(scale_f), N.ptr(shift_f),
                                                      N.ptr(out), m, out_features, k, group_size,
                                                      N.DTYPE_CODE[gO.dtype], shift_is_int, N.stream_ptr(gO.device)),
                        "quanto::qbits_grad_input")
                return out
            except N.UnsupportedConfiguration:
                pass
    w = dequantize_qbits_cuda(packed, scale, shift, out_features, k, group_size, bits)
    return torch.matmul(gO, w)


def _check_qbytes_grad_input(grad_output, weights, scales):
    if weights.ndim != 2:
        raise ValueError("qbytes_grad_input expects weights [N, K]")
    if weights.dtype not in (torch.int8, torch.float8_e4m3fn, torch.float8_e5m2, torch.float8_e4m3fnuz):
        raise NotImplementedError(f"qbytes_grad_input: no sm_90a kernel for weights of dtype {weights.dtype}")
    n = weights.shape[0]
    _check_grad_output_2d(grad_output, n, "qbytes_grad_input")
    if grad_output.dtype != scales.dtype or scales.dtype not in _FLOATS:
        raise ValueError(f"qbytes_grad_input: grad_output dtype {grad_output.dtype} does not match the scales "
                         f"({scales.dtype})")
    if scales.numel() != n and scales.numel() != 1:
        raise ValueError("qbytes_grad_input: scales must have one value per output feature or one in all")


def qbytes_grad_input_cuda(grad_output, weights, scales):
    """dX = gO @ (scales * W) for an 8-bit weight [N, K] with per-out-feature scales: ONE native launch.

    Shapes the kernel declines (fp32, per-tensor scale, N % 8 != 0, K % 16 != 0, unaligned buffers) run the composition
    the reference's backward performs: `scales * W` in the scale dtype (QBytesDequantizer), then matmul."""
    _check_qbytes_grad_input(grad_output, weights, scales)
    n, k = weights.shape
    gO = _require_contiguous(grad_output, "grad_output")
    if scales.numel() == n and n > 1:
        m = gO.shape[0]
        w = _require_contiguous(weights, "B")
        s = _require_contiguous(scales.reshape(-1), "scales")
        out = torch.empty((m, k), dtype=gO.dtype, device=gO.device)
        with torch.cuda.device(gO.device):
            lib = N.load()
            try:
                N.check(lib.qb200_qbytes_mm_grad_input(N.ptr(gO), N.ptr(w), N.ptr(s), N.ptr(out), m, n, k,
                                                       N.DTYPE_CODE[w.dtype], N.DTYPE_CODE[gO.dtype],
                                                       N.stream_ptr(gO.device)), "quanto::qbytes_grad_input")
                return out
            except N.UnsupportedConfiguration:
                pass
    payload = weights.to(scales.dtype) if weights.dtype.is_floating_point else weights  # fp8 has no mul
    scale_b = scales.reshape(-1, 1) if scales.numel() == n else scales
    return torch.matmul(gO, scale_b * payload)


def _bind_cuda(name: str, fn):
    """Attach the sm_90a implementation to the CUDA dispatch key, replacing the reference's CUDA binding if
    `optimum.quanto` was imported first (it registers its own for unpack / qbytes_mm,
    optimum/quanto/library/extensions/cuda/__init__.py:77-79, library/qbytes_mm.py:73)."""
    _lib.impl(name, fn, "CUDA", allow_override=True)


_bind_cuda("unpack", unpack_cuda)
_bind_cuda("quantize_symmetric", quantize_symmetric_cuda)
_bind_cuda("qbytes_mm", _qbytes_mm_op)
_bind_cuda("qbytes_linear", _qbytes_linear_op)
_bind_cuda("qbytes_linear_quantized", qbytes_linear_quantized_cuda)
_bind_cuda("qbits_mm", qbits_mm_cuda)
_bind_cuda("dequantize_qbits", dequantize_qbits_cuda)
_bind_cuda("qbits_grad_input", qbits_grad_input_cuda)
_bind_cuda("qbytes_grad_input", qbytes_grad_input_cuda)
_bind_cuda("pack", pack_cuda)
_bind_cuda("quantize_qbits_max", quantize_qbits_max_cuda)
_bind_cuda("quantize_qbytes_absmax", quantize_qbytes_absmax_cuda)
_bind_cuda("absmax", absmax_cuda)
_bind_cuda("quantize_qbits_hqq", quantize_qbits_hqq_cuda)
_bind_cuda("hqq_shrink", hqq_shrink_cuda)
_bind_cuda("quantize_affine", quantize_affine_cuda)
try:
    _lib.impl("quantize_affine", quantize_affine_any, "CompositeExplicitAutograd")
except RuntimeError:
    pass  # the reference package already bound its own python implementation


# ------------------------------------------------------------------------------------------ fake implementations
# What FakeTensor tracing (torch.compile, AOTAutograd) sees of each op: the output metadata the CUDA implementation above
# allocates, after the same argument checks.  Sizes may be SymInts, so the token count M can stay dynamic.
def _unpack_fake(packed, bits):
    return packed.new_empty(_unpack_shape(packed, bits), dtype=torch.uint8)


def _quantize_symmetric_fake(base, dtype, axis, scale):
    _quantize_symmetric_plan(base, dtype, axis, scale)
    return base.new_empty(base.shape, dtype=dtype)


def _quantize_affine_fake(base, bits, axis, group_size, scale, shift):
    grouped, mode = _quantize_affine_plan(base, bits, axis, group_size, scale, shift)
    if mode is None or not grouped.is_cuda:
        return _quantize_affine_aten(grouped, bits, scale, shift)
    return grouped.new_empty(grouped.shape, dtype=torch.uint8)


def _pack_fake(values, bits):
    return values.new_empty(_pack_shape(values, bits), dtype=torch.uint8)


def _quantize_qbits_max_fake(base, bits, group_size, zeropoint):
    packed_shape, coef_shape, shift_dtype = _freeze_qbits_shapes("quantize_qbits_max", base, bits, group_size, zeropoint)
    return (base.new_empty(packed_shape, dtype=torch.uint8), base.new_empty(coef_shape),
            base.new_empty(coef_shape, dtype=shift_dtype))


def _quantize_qbits_hqq_fake(base, bits, group_size, zeropoint, lp_norm, beta, kappa, iters):
    packed_shape, coef_shape, shift_dtype = _freeze_qbits_shapes("quantize_qbits_hqq", base, bits, group_size, zeropoint)
    return (base.new_empty(packed_shape, dtype=torch.uint8), base.new_empty(coef_shape),
            base.new_empty(coef_shape, dtype=shift_dtype), base.new_empty((max(iters, 0) + 2,), dtype=torch.float32))


def _hqq_shrink_fake(x, beta, lp_norm):
    _check_float("hqq_shrink", x)
    return x.new_empty(x.shape)


def _quantize_qbytes_absmax_fake(base, dtype):
    _check_qbytes_absmax(base, dtype)
    n, k = base.shape
    return base.new_empty((n, k), dtype=dtype), base.new_empty((n, 1))


def _absmax_fake(base):
    _check_float("absmax", base)
    return base.new_empty(())


def _qbytes_mm_fake(activations, weights, output_scales):
    _check_qbytes_mm(activations, weights, output_scales)
    return activations.new_empty(activations.shape[:-1] + (weights.shape[0],), dtype=output_scales.dtype)


def _qbytes_linear_fake(activations, weights, output_scales, bias):
    out = _qbytes_mm_fake(activations, weights, output_scales)
    if bias is not None and not _bias_in_epilogue(weights, output_scales, bias):
        return out + bias
    return out


def _qbytes_linear_quantized_fake(activations, weights, output_scales, bias, out_scale, out_dtype):
    if _qbytes_linear_quantized_fusable(activations, weights, output_scales, bias, out_scale, out_dtype):
        return activations.new_empty(activations.shape[:-1] + (weights.shape[0],), dtype=out_dtype)
    y = _qbytes_linear_fake(activations, weights, output_scales, bias)
    return _quantize_symmetric_fake(y, out_dtype, None, out_scale.reshape(()))


def _dequantize_qbits_fake(packed, scale, shift, out_features, in_features, group_size, bits):
    _check_dequantize_qbits(shift)
    return packed.new_empty((out_features, in_features), dtype=scale.dtype)


def _qbits_mm_fake(activations, packed, scale, shift, bias, out_features, group_size, bits=4):
    _check_qbits_mm(activations, packed, scale, shift, bias, out_features, group_size, bits)
    return activations.new_empty(activations.shape[:-1] + (out_features,))


def _qbits_grad_input_fake(grad_output, packed, scale, shift, out_features, group_size, bits):
    k = _check_qbits_grad_input(grad_output, packed, scale, shift, out_features, group_size, bits)
    return grad_output.new_empty((grad_output.shape[0], k))


def _qbytes_grad_input_fake(grad_output, weights, scales):
    _check_qbytes_grad_input(grad_output, weights, scales)
    return grad_output.new_empty((grad_output.shape[0], weights.shape[1]))


FAKE_IMPLS = {
    "unpack": _unpack_fake,
    "qbytes_mm": _qbytes_mm_fake,
    "quantize_symmetric": _quantize_symmetric_fake,
    "quantize_affine": _quantize_affine_fake,
    "qbits_mm": _qbits_mm_fake,
    "dequantize_qbits": _dequantize_qbits_fake,
    "qbytes_linear": _qbytes_linear_fake,
    "qbytes_linear_quantized": _qbytes_linear_quantized_fake,
    "pack": _pack_fake,
    "quantize_qbits_max": _quantize_qbits_max_fake,
    "quantize_qbytes_absmax": _quantize_qbytes_absmax_fake,
    "absmax": _absmax_fake,
    "quantize_qbits_hqq": _quantize_qbits_hqq_fake,
    "hqq_shrink": _hqq_shrink_fake,
    "qbits_grad_input": _qbits_grad_input_fake,
    "qbytes_grad_input": _qbytes_grad_input_fake,
}
for _name, _fake in FAKE_IMPLS.items():
    torch.library.register_fake("quanto::" + _name, _fake, lib=_lib)
