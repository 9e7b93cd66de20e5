"""The aten op table of per-tensor quantized activations (optimum/quanto/tensor/activations/qbytes_ops.py).

Layout ops, copies and joins act on `_data` and keep `_scale`, so that a QLinear's quantized output stays quantized
through the view / transpose / permute / expand / clone of an attention block; scalar `div` / `mul` only touch the
scale; `bmm` of two qint8 activations and `_softmax` over the last dim run on the library's kernels
(`quanto::qbytes_bmm`, `quanto::qbytes_softmax`).  Every op outside the table, `bmm` with a float first operand and
float8 arithmetic dequantize, as in the reference.

Two entries port what the reference means rather than what it does: its `stack` fallback calls `qfallback(inputs, dim)`
without the op, and its `clone` reshapes the data to the outer shape and then clones the un-reshaped data
(qbytes_ops.py:108-117, 218-233).
"""
import numbers

import torch

from .activations import ActivationQBytesTensor, quantize_activation
from .core import dtype_info
from .qtensor import QTensor, qfallback
from .qtype import qint8

__all__ = ["get_qbytestensor_op_dispatch"]

aten = torch.ops.aten
_OP_TABLE = {}


def _register(aten_ops):
    def wrapper(fn):
        for aten_op in aten_ops:
            _OP_TABLE[aten_op] = (fn, aten_op)
        return fn

    return wrapper


def get_qbytestensor_op_dispatch(packet):
    """The table entry of an aten overload packet as a callable of (*args, **kwargs), or None."""
    entry = _OP_TABLE.get(packet)
    if entry is None:
        return None
    fn, op = entry
    return lambda *args, **kwargs: fn(op, *args, **kwargs)


def _is_scalar(t):
    return isinstance(t, numbers.Number) or type(t) is torch.Tensor and len(t.shape) == 0


def _wrap(qtype, data, scale):
    return ActivationQBytesTensor(qtype, data.size(), data.stride(), data, scale)


@_register([aten._to_copy, aten.to])
def _to_copy(op, t, **kwargs):
    dtype = kwargs.pop("dtype", t.dtype)
    if dtype is not None and dtype != t.dtype:
        raise ValueError("The dtype of an activations Tensor cannot be changed")
    return ActivationQBytesTensor(t.qtype, t.size(), t.stride(), op(t._data, **kwargs), op(t._scale, **kwargs))


@_register([aten.detach])
def detach(op, t):
    return ActivationQBytesTensor(t.qtype, t.size(), t.stride(), op(t._data), op(t._scale))


def _same_scale(t1, t2):
    return (isinstance(t1, ActivationQBytesTensor) and isinstance(t2, ActivationQBytesTensor)
            and t1.qtype == t2.qtype and torch.equal(t1._scale, t2._scale))


@_register([aten.cat])
def cat(op, inputs, dim=0):
    if len(inputs) == 2 and _same_scale(*inputs) and not inputs[0].qtype.is_floating_point:
        return _wrap(inputs[0].qtype, op([inputs[0]._data, inputs[1]._data], dim), inputs[0]._scale)
    return qfallback(op, inputs, dim)


@_register([aten.stack])
def stack(op, inputs, dim=0):
    if len(inputs) == 2 and _same_scale(*inputs) and inputs[0].axis is None and inputs[1].axis is None:
        return _wrap(inputs[0].qtype, op([inputs[0]._data, inputs[1]._data], dim), inputs[0]._scale)
    return qfallback(op, inputs, dim)


@_register([aten.lt])
def lt(op, input, other):
    if isinstance(input, ActivationQBytesTensor) and isinstance(other, ActivationQBytesTensor) and torch.equal(
            input._scale, other._scale):
        return op(input._data, other._data)
    return qfallback(op, input, other)


@_register([aten.clone])
def clone(op, t, memory_format=torch.preserve_format):
    # clone the data in the outer shape, so that the clone's strides are those of the outer tensor
    data_shape = t._data.shape
    out_data = op(t._data.reshape(t.shape), memory_format=memory_format)
    out_stride = out_data.stride()
    out_data = out_data.reshape(data_shape)
    return ActivationQBytesTensor(t.qtype, t.size(), out_stride, out_data, op(t._scale, memory_format=memory_format))


@_register([aten.copy_])
def copy_(op, dest, src):
    assert dest.qtype == src.qtype
    dest._data = op(dest._data, src._data)
    dest._scale = op(dest._scale, src._scale)
    return dest


@_register([aten.div])
def div(op, input, other):
    if not _is_scalar(other):
        return op(input.dequantize(), other)
    return ActivationQBytesTensor(input.qtype, input.size(), input.stride(), input._data, op(input._scale, other))


@_register([aten.mul])
def mul(op, input, other):
    if _is_scalar(input):
        return ActivationQBytesTensor(other.qtype, other.size(), other.stride(), other._data, input * other._scale)
    if _is_scalar(other):
        return ActivationQBytesTensor(input.qtype, input.size(), input.stride(), input._data, other * input._scale)
    return qfallback(op, input, other)


@_register([aten.neg])
def neg(op, input, *args, **kwargs):
    if input.qtype.is_floating_point:
        return op(input.dequantize(), *args, **kwargs)
    return ActivationQBytesTensor(input.qtype, input.size(), input.stride(), op(input._data, *args, **kwargs),
                                  input._scale)


@_register([aten.relu])
def relu(op, input):
    if input.qtype.is_floating_point:
        return qfallback(op, input)
    return ActivationQBytesTensor(input.qtype, input.size(), input.stride(), op(input._data), input._scale)


@_register([aten.expand, aten.permute, aten.select, aten.slice, aten.unsqueeze])
def unary_type_agnostic_op(op, input, *args, **kwargs):
    if input.axis is not None:
        return op(input.dequantize(), *args, **kwargs)
    return _wrap(input.qtype, op(input._data, *args, **kwargs), input._scale)


@_register([aten.is_same_size])
def is_same_size(op, input, other):
    a = input._data if isinstance(input, ActivationQBytesTensor) else input
    b = other._data if isinstance(other, ActivationQBytesTensor) else other
    return op(a, b)


def _cannot_mm(t: QTensor):
    return t.axis is not None and t.size() != t._data.size()


@_register([aten.bmm])
def bmm(op, input, other):
    if not isinstance(input, ActivationQBytesTensor):
        return op(input, other.dequantize())
    if not isinstance(other, QTensor) or input.axis is not None:
        return op(input.dequantize(), other)
    if input.qtype != qint8 or other.qtype != qint8 or _cannot_mm(other):
        return qfallback(op, input, other)
    if other._scale.numel() != 1 or other._scale.dtype != input._scale.dtype:
        return qfallback(op, input, other)  # a per-axis or differently typed scale: no kernel takes it
    return torch.ops.quanto.qbytes_bmm(input._data, other._data, input._scale, other._scale)


@_register([aten._softmax])
def _softmax(op, input, dim, half_to_float):
    # softmax is normalised, so the output scale is known: 1 / qmax
    out_scale = torch.tensor(1 / dtype_info(input.qtype.dtype).max, dtype=input._scale.dtype).to(input.device)
    if input.axis is None and not half_to_float and dim in (-1, input.ndim - 1):
        data = torch.ops.quanto.qbytes_softmax(input._data, input._scale, out_scale)
        return _wrap(input.qtype, data, out_scale)
    float_data = op(input.dequantize(), dim, half_to_float)
    return quantize_activation(float_data, qtype=input.qtype, scale=out_scale)


@_register([aten.split])
def split(op, input, *args, **kwargs):
    if input.axis is not None:
        return qfallback(op, input, *args, **kwargs)
    return [_wrap(input.qtype, out_data, input._scale) for out_data in op(input._data, *args, **kwargs)]


@_register([aten.transpose])
def transpose(op, input, *args):
    return _wrap(input.qtype, op(input._data, *args), input._scale)


@_register([aten.t])
def transpose2d(op, input):
    out_data = op(input._data)
    dim0, dim1 = input.size()
    return ActivationQBytesTensor(input.qtype, torch.Size([dim1, dim0]), input.stride()[::-1], out_data, input._scale)


@_register([aten.view, aten._unsafe_view])
def view(op, input, *shape):
    if input.axis is None:
        return _wrap(input.qtype, op(input._data, *shape), input._scale)
    return qfallback(op, input, *shape)


@_register([aten.where])
def where(op, condition, input, other):
    if isinstance(condition, QTensor) or isinstance(other, QTensor):
        raise NotImplementedError
    float_data = op(condition, input.dequantize(), other)
    if input.axis is None:
        return quantize_activation(float_data, qtype=input.qtype, scale=input._scale)
    return float_data
