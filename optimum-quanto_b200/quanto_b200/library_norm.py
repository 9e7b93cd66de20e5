"""`quanto::qbytes_layer_norm`: the reference's QLayerNorm (optimum/quanto/nn/qlayernorm.py:27-53) as one launch.

The reference runs F.layer_norm (after qfallback dequantizes an ActivationQBytesTensor input, tensor/qbytes.py:23-31)
and then the quantize_output hook (nn/qmodule.py:296-302 -> quanto::quantize_symmetric): two or three launches with the
[rows, H] activation written and read back in 16 or 32 bits in between.  This op reads the input once (floats or 8-bit
codes) and writes the output once (8-bit codes, or floats when no output scale is given).

`qlayernorm_forward` is the one place that decides when a QLayerNorm takes the op; the package's QLayerNorm and
`integration.bind_reference()` both call it.  Defined here rather than in library.py so that each module registers and
fakes exactly the ops it defines.
"""
import math

import torch

from . import _native as N
from .library import _FLOATS, _bind_cuda, _define, _lib

__all__ = []

_define("qbytes_layer_norm", "(Tensor input, Tensor? input_scale, int[] normalized_shape, Tensor? weight, Tensor? bias, "
                             "float eps, Tensor? output_scale, ScalarType? output_dtype) -> Tensor")

_CODES = (torch.int8, torch.float8_e4m3fn, torch.float8_e5m2, torch.float8_e4m3fnuz)


def _check_qbytes_layer_norm(input, input_scale, normalized_shape, weight, bias, output_scale, output_dtype):
    """The argument checks of quanto::qbytes_layer_norm -> (float dtype T, output dtype, H)."""
    shape = tuple(normalized_shape)
    if len(shape) == 0 or input.ndim < len(shape) or tuple(input.shape[input.ndim - len(shape):]) != shape:
        raise ValueError(f"qbytes_layer_norm: normalized_shape {list(shape)} does not end the input shape "
                         f"{list(input.shape)}")
    if input_scale is not None:
        if input.dtype not in _CODES:
            raise ValueError(f"qbytes_layer_norm: an input with a scale must be 8-bit codes (got {input.dtype})")
        if input_scale.dtype not in _FLOATS or input_scale.numel() != 1:
            raise ValueError("qbytes_layer_norm: the input scale must be one floating point element")
        dtype = input_scale.dtype
    else:
        if input.dtype not in _FLOATS:
            raise ValueError(f"qbytes_layer_norm: a float input must be float32, float16 or bfloat16 (got {input.dtype})")
        dtype = input.dtype
    for name, p in (("weight", weight), ("bias", bias)):
        if p is not None and (p.dtype != dtype or tuple(p.shape) != shape):
            raise ValueError(f"qbytes_layer_norm: {name} must be {list(shape)} in {dtype} (got {list(p.shape)} "
                             f"{p.dtype})")
    if output_scale is not None:
        if output_dtype not in _CODES:
            raise ValueError(f"qbytes_layer_norm: output dtype {output_dtype} is not an 8-bit code dtype")
        if output_scale.numel() != 1 or output_scale.dtype not in (torch.float32, dtype):
            raise ValueError(f"qbytes_layer_norm: the output scale must be one float32 or {dtype} element")
        out_dtype = output_dtype
    else:
        if output_dtype is not None:
            raise ValueError("qbytes_layer_norm: an output dtype needs an output scale")
        out_dtype = dtype
    for name, t in (("input_scale", input_scale), ("weight", weight), ("bias", bias), ("output_scale", output_scale)):
        if t is not None and t.device != input.device:
            raise ValueError(f"qbytes_layer_norm: {name} is on {t.device}, the input on {input.device}")
    return dtype, out_dtype, math.prod(shape)


def qbytes_layer_norm_cuda(input, input_scale, normalized_shape, weight, bias, eps, output_scale, output_dtype):
    """quantize_symmetric(F.layer_norm(dequantize(input), ...), output_dtype, None, output_scale) in one launch."""
    dtype, out_dtype, h = _check_qbytes_layer_norm(input, input_scale, normalized_shape, weight, bias, output_scale,
                                                   output_dtype)
    x = input.contiguous()
    out = torch.empty(x.shape, dtype=out_dtype, device=x.device)
    if x.numel() == 0:
        return out
    rows = x.numel() // h
    flat = [None if t is None else t.reshape(-1).contiguous() for t in (input_scale, weight, bias, output_scale)]
    with torch.cuda.device(x.device):
        lib = N.load()
        N.check(lib.qb200_layer_norm(N.ptr(x), *(N.ptr(t) for t in flat), N.ptr(out), rows, h, float(eps),
                                     N.DTYPE_CODE[x.dtype], N.DTYPE_CODE[dtype], N.DTYPE_CODE[out_dtype],
                                     N.DTYPE_CODE[output_scale.dtype] if output_scale is not None else N.F32,
                                     N.stream_ptr(x.device)), "quanto::qbytes_layer_norm")
    return out


_bind_cuda("qbytes_layer_norm", qbytes_layer_norm_cuda)


def _qbytes_layer_norm_fake(input, input_scale, normalized_shape, weight, bias, eps, output_scale, output_dtype):
    _, out_dtype, _ = _check_qbytes_layer_norm(input, input_scale, normalized_shape, weight, bias, output_scale,
                                               output_dtype)
    return input.new_empty(input.shape, dtype=out_dtype)


FAKE_IMPLS = {"qbytes_layer_norm": _qbytes_layer_norm_fake}
for _name, _fake in FAKE_IMPLS.items():
    torch.library.register_fake("quanto::" + _name, _fake, lib=_lib)


# ------------------------------------------------------------------------------------------ module routing
def qlayernorm_forward(module, input, activation_cls, output_hook_live: bool):
    """The forward of a QLayerNorm `module` as one `quanto::qbytes_layer_norm` launch, or None when F.layer_norm has to
    run instead.

    Taken when no gradient is needed, the weight and bias are absent or in the float dtype T of the input (a CUDA float
    tensor, or a per-tensor `activation_cls` whose scale dtype is T), and the scales are on the input's device.  With the
    output hook live it returns an `activation_cls` of the module's activation qtype over the op's codes and
    `module.output_scale` (the hook then has nothing left to quantize); with the hook removed, a codes input gives the
    op's float output and a float input keeps F.layer_norm.  `output_hook_live` says whether the module's
    quantize_output hook is registered."""
    weight, bias = module.weight, module.bias
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (input, weight, bias)):
        return None
    if isinstance(input, activation_cls):
        data, scale = input._data, input._scale
        if input.axis is not None or scale.numel() != 1 or data.dtype not in _CODES:
            return None
        dtype = scale.dtype
    else:
        if type(input) is not torch.Tensor:
            return None
        data, scale, dtype = input, None, input.dtype
    if not data.is_cuda or dtype not in _FLOATS or (scale is not None and scale.device != data.device):
        return None
    if any(p is not None and (p.dtype != dtype or p.device != data.device) for p in (weight, bias)):
        return None
    if output_hook_live:
        qtype, out_scale = module.activation_qtype, module.output_scale
        if out_scale.device != data.device or out_scale.dtype not in (torch.float32, dtype) or out_scale.numel() != 1:
            return None
        codes = torch.ops.quanto.qbytes_layer_norm(data, scale, list(module.normalized_shape), weight, bias,
                                                   module.eps, out_scale, qtype.dtype)
        return activation_cls(qtype, codes.size(), codes.stride(), codes, out_scale)
    if scale is None:
        return None
    return torch.ops.quanto.qbytes_layer_norm(data, scale, list(module.normalized_shape), weight, bias, module.eps,
                                              None, None)
