"""Weight QTensors: `WeightQBytesTensor` (int8 / float8) and `WeightQBitsTensor` (int4 / int2).

Same constructor signatures, factory names, serialization keys and torch-function/dispatch hooks as
optimum/quanto/tensor/weights/qbytes.py:31-326 and optimum/quanto/tensor/weights/qbits.py:34-317.  The difference
is in `create()`: there is no kernel-specific repacking any more (AWQ / Marlin / TinyGemm subclasses are gone); the
The kernels read quanto's canonical storage directly, so `create()` always returns the canonical class and
`optimize()` is the identity.
"""
import ast
from typing import Optional

import torch
from torch.autograd import Function

from .function import QuantizedLinearFunction, WeightQBitsLinearFunction, WeightQBytesLinearFunction
from .grouped import grouped_shape
from .packed import PackedTensor
from .qtensor import QBitsTensor, QBytesTensor, qfallback
from .qtype import qint2, qint4, qtype, qtypes

__all__ = ["WeightQBytesTensor", "WeightQBitsTensor", "quantize_weight"]


# ------------------------------------------------------------------------------------------- 8 bit
class WeightQBytesQuantizer(Function):
    @staticmethod
    def forward(ctx, base, qtype, axis, scale, activation_qtype, optimized):
        if qtype.bits != 8:
            raise ValueError("QBytesTensor can only be of 8-bit qtype")
        data = torch.ops.quanto.quantize_symmetric(base, dtype=qtype.dtype, axis=axis, scale=scale)
        make = WeightQBytesTensor.create if optimized else WeightQBytesTensor
        return make(qtype, axis, size=base.size(), stride=base.stride(), data=data, scale=scale,
                    activation_qtype=activation_qtype)

    @staticmethod
    def backward(ctx, gO):
        return gO, None, None, None, None, None, None


class WeightQBytesTensor(QBytesTensor):
    @staticmethod
    def create(qtype, axis, size, stride, data, scale, activation_qtype: Optional[qtype] = None, requires_grad=False):
        """Factory kept for API compatibility; the canonical tensor is already the optimal one on H100."""
        return WeightQBytesTensor(qtype, axis, size, stride, data, scale, activation_qtype, requires_grad)

    @staticmethod
    def __new__(cls, qtype, axis, size, stride, data, scale, activation_qtype, requires_grad=False):
        assert data.device == scale.device
        return torch.Tensor._make_wrapper_subclass(
            cls, size, strides=stride, dtype=scale.dtype, device=data.device, requires_grad=requires_grad
        )

    def __init__(self, qtype, axis, size, stride, data, scale, activation_qtype, requires_grad=False):
        super().__init__(qtype, axis, size, stride, data, scale, requires_grad=requires_grad)
        self.activation_qtype = activation_qtype

    @classmethod
    def quantize(cls, base, qtype, axis, scale, activation_qtype=None, optimized=True):
        return WeightQBytesQuantizer.apply(base, qtype, axis, scale, activation_qtype, optimized)

    @staticmethod
    def load_from_state_dict(state_dict, prefix, qtype, axis, size, stride, activation_qtype, missing_keys):
        inner = {}
        for name in ("_data", "_scale"):
            if prefix + name not in state_dict:
                missing_keys.append(prefix + name)
            else:
                inner[name] = state_dict.pop(prefix + name)
        if len(inner) != 2:
            return None
        meta = {
            "qtype": qtype.name,
            "axis": str(axis),
            "size": str(list(size)),
            "stride": str(list(stride)),
            "activation_qtype": "none" if activation_qtype is None else activation_qtype.name,
        }
        return WeightQBytesTensor.__tensor_unflatten__(inner, meta, None, None)

    def optimize(self):
        return self

    def weight_qbytes_tensor(self):
        return self

    def __tensor_flatten__(self):
        meta = {
            "qtype": self._qtype.name,
            "axis": str(self._axis),
            "size": str(list(self.size())),
            "stride": str(list(self.stride())),
            "activation_qtype": "none" if self.activation_qtype is None else self.activation_qtype.name,
        }
        return ["_data", "_scale"], meta

    @staticmethod
    def __tensor_unflatten__(inner_tensors, meta, outer_size, outer_stride):
        assert len(inner_tensors) == 2 and len(meta) == 5
        act = None if meta["activation_qtype"] == "none" else qtypes[meta["activation_qtype"]]
        return WeightQBytesTensor(
            qtypes[meta["qtype"]],
            ast.literal_eval(meta["axis"]),
            ast.literal_eval(meta["size"]),
            ast.literal_eval(meta["stride"]),
            inner_tensors["_data"],
            inner_tensors["_scale"],
            act,
        )

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func is torch.nn.functional.linear:
            return WeightQBytesLinearFunction.apply(*_linear_args(*args, **kwargs))
        if func is torch.nn.functional.conv2d:
            out = _native_conv2d(args, kwargs)
            if out is not None:
                return out
        if func is torch.equal:
            return args[0].equal(args[1])
        with torch._C.DisableTorchFunctionSubclass():
            return func(*args, **kwargs)

    @classmethod
    def __torch_dispatch__(cls, op, types, args, kwargs=None):
        kwargs = dict(kwargs or {})
        packet = op.overloadpacket
        if packet is torch.ops.aten.detach:
            t = args[0]
            names, meta = t.__tensor_flatten__()
            return cls.__tensor_unflatten__({n: packet(getattr(t, n)) for n in names}, meta, t.size(), t.stride())
        if packet in (torch.ops.aten._to_copy, torch.ops.aten.to):
            t = args[0]
            dtype = kwargs.pop("dtype", t.dtype)
            device = kwargs.pop("device", t.device)
            if dtype is not None and dtype != t.dtype:
                raise ValueError("The dtype of a weights Tensor cannot be changed")
            data = packet(t._data, device=device, **kwargs)
            scale = packet(t._scale, device=device, **kwargs)
            return WeightQBytesTensor.create(t.qtype, t.axis, t.size(), t.stride(), data, scale,
                                             activation_qtype=t.activation_qtype, requires_grad=t.requires_grad)
        if packet is torch.ops.aten.t and cls is WeightQBytesTensor:
            t = args[0]
            scale, axis = t._scale, t.axis
            rows, cols = t.size()
            if axis is not None:
                scale = packet(scale)
                axis = 0 if axis == -1 else -1
            return WeightQBytesTensor(t.qtype, axis, torch.Size([cols, rows]), t.stride()[::-1], packet(t._data),
                                      scale, t.activation_qtype)
        return qfallback(packet, *args, **kwargs)


# --------------------------------------------------------------------------------------- 4 / 2 bit
class WeightsQBitsQuantizer(Function):
    @staticmethod
    def forward(ctx, base, qtype, axis, group_size, scale, shift, optimized):
        if qtype not in (qint2, qint4):
            raise ValueError("WeightQBitsTensor can only be of qint2 or qint4 qtype")
        if axis not in (0, -1):
            raise ValueError("WeightQBitsTensor axis parameter must be 0 (first axis) or -1 (last axis)")
        data = torch.ops.quanto.quantize_affine(base, bits=qtype.bits, axis=axis, group_size=group_size, scale=scale,
                                                shift=shift)
        make = WeightQBitsTensor.create if optimized else WeightQBitsTensor
        return make(qtype, axis, group_size, base.size(), base.stride(), data, scale, shift)

    @staticmethod
    def backward(ctx, gO):
        return gO, None, None, None, None, None, None


class WeightQBitsTensor(QBitsTensor):
    @staticmethod
    def create(qtype, axis, group_size, size, stride, data, scale, shift, requires_grad=False):
        """No AWQ / TinyGemm routing: the fused sm_90a kernel consumes the canonical packing as is."""
        return WeightQBitsTensor(qtype, axis, group_size, size, stride, data, scale, shift, requires_grad)

    @staticmethod
    def __new__(cls, qtype, axis, group_size, size, stride, data, scale, shift, requires_grad=False):
        assert data.device == scale.device
        assert data.device == shift.device
        return torch.Tensor._make_wrapper_subclass(
            cls, size, strides=stride, dtype=scale.dtype, device=data.device, requires_grad=requires_grad
        )

    def __init__(self, qtype, axis, group_size, size, stride, data, scale, shift, requires_grad=False):
        if type(data) is torch.Tensor:
            data = PackedTensor.pack(data, qtype.bits)
        super().__init__(qtype, axis, group_size, size, stride, data, scale, shift)

    @classmethod
    def quantize(cls, base, qtype, axis, group_size, scale, shift, optimized=True):
        return WeightsQBitsQuantizer.apply(base, qtype, axis, group_size, scale, shift, optimized)

    @staticmethod
    def load_from_state_dict(state_dict, prefix, qtype, axis, group_size, size, stride, missing_keys):
        if group_size is None:
            data_size, data_stride = size, stride
        else:
            data_size = grouped_shape(size, axis, group_size)
            data_stride = (data_size[1], 1)
        inner = {"_data": PackedTensor.load_from_state_dict(state_dict, prefix + "_data.", qtype.bits, data_size,
                                                            data_stride, missing_keys=missing_keys)}
        missing = inner["_data"] is None
        for name in ("_scale", "_shift"):
            if prefix + name not in state_dict:
                missing_keys.append(prefix + name)
                missing = True
            else:
                inner[name] = state_dict.pop(prefix + name)
        if missing:
            return None
        meta = {
            "qtype": qtype.name,
            "axis": str(axis),
            "group_size": str(group_size),
            "size": str(list(size)),
            "stride": str(list(stride)),
        }
        return WeightQBitsTensor.__tensor_unflatten__(inner, meta, None, None)

    def optimize(self):
        return self

    def weight_qbits_tensor(self):
        return self

    def __tensor_flatten__(self):
        meta = {
            "qtype": self._qtype.name,
            "axis": str(self._axis),
            "group_size": str(self._group_size),
            "size": str(list(self.size())),
            "stride": str(list(self.stride())),
        }
        return ["_data", "_scale", "_shift"], meta

    @staticmethod
    def __tensor_unflatten__(inner_tensors, meta, outer_size, outer_stride):
        assert len(inner_tensors) == 3 and len(meta) == 5
        return WeightQBitsTensor(
            qtypes[meta["qtype"]],
            ast.literal_eval(meta["axis"]),
            ast.literal_eval(meta["group_size"]),
            ast.literal_eval(meta["size"]),
            ast.literal_eval(meta["stride"]),
            inner_tensors["_data"],
            inner_tensors["_scale"],
            inner_tensors["_shift"],
        )

    def _fused_linear_ok(self, input) -> bool:
        """Configurations `quanto::qbits_mm` takes in one native launch: any axis-0 packed int4 / int2 weight on a CUDA
        device whose float dtype matches the activations (grouped or per-axis, float shift or zero-point).  Only axis -1
        quantisation -- never produced for a linear weight (nn/qmodule.py quantizes along axis 0) -- dequantises first.

        Autograd does not matter here: the backward of the fused forward is explicit (function.py).
        """
        if len(self.shape) != 2 or not isinstance(self._data, PackedTensor):
            return False
        n, k = self.shape
        g = self._group_size if self._group_size is not None else k
        shift_ok = (self._shift.dtype in (torch.uint8, torch.int8)) or self._shift.dtype == self._scale.dtype
        in_dtype = input._scale.dtype if isinstance(input, QBytesTensor) else input.dtype
        return (
            self._qtype.bits in (2, 4) and not self._qtype.is_floating_point
            and self._axis == 0
            and self._data._data.is_cuda
            and self._scale.dtype in (torch.float32, torch.float16, torch.bfloat16)
            and shift_ok
            and g > 0 and k % g == 0
            and self._scale.numel() == n * (k // g)
            and in_dtype == self._scale.dtype
        )

    @classmethod
    def __torch_function__(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func is torch.nn.functional.linear:
            input, other, bias = _linear_args(*args, **kwargs)
            if isinstance(other, WeightQBitsTensor) and other._fused_linear_ok(input):
                return WeightQBitsLinearFunction.apply(input, other, bias)
            return QuantizedLinearFunction.apply(input, other, bias)
        if func is torch.nn.functional.conv2d:
            out = _native_conv2d(args, kwargs)
            if out is not None:
                return out
        if func is torch.equal:
            return args[0].equal(args[1])
        with torch._C.DisableTorchFunctionSubclass():
            return func(*args, **kwargs)

    @classmethod
    def __torch_dispatch__(cls, op, types, args, kwargs=None):
        kwargs = dict(kwargs or {})
        packet = op.overloadpacket
        if packet is torch.ops.aten.detach:
            t = args[0]
            names, meta = t.__tensor_flatten__()
            return cls.__tensor_unflatten__({n: packet(getattr(t, n)) for n in names}, meta, t.size(), t.stride())
        if packet in (torch.ops.aten._to_copy, torch.ops.aten.to):
            t = args[0]
            dtype = kwargs.pop("dtype", t.dtype)
            device = kwargs.pop("device", t.device)
            if dtype is not None and dtype != t.dtype:
                raise ValueError("The dtype of a WeightQBitsTensor cannot be changed")
            scale = packet(t._scale, dtype=dtype, device=device, **kwargs)
            data = packet(t._data, device=device, **kwargs)
            shift = packet(t._shift, device=device, **kwargs)
            return WeightQBitsTensor.create(t._qtype, t._axis, t._group_size, t.size(), t.stride(), data, scale, shift)
        return qfallback(packet, *args, **kwargs)


def _linear_args(input, weight=None, bias=None, **kw):
    if weight is None:
        weight = kw["weight"]
    if "bias" in kw:
        bias = kw["bias"]
    return input, weight, bias


def _native_conv2d(args, kwargs):
    """F.conv2d on a quantized weight as one quanto::qbits_conv2d / quanto::qbytes_conv2d launch, or None: the caller then
    runs the reference's composition (library_conv.native_conv2d)."""
    from .. import library_conv

    return library_conv.native_conv2d(args, kwargs, WeightQBitsTensor, WeightQBytesTensor)


def quantize_weight(t, qtype, axis, scale, shift=None, group_size=None, activation_qtype=None, optimized=True):
    """Quantize a weight tensor per-axis (optimum/quanto/tensor/weights/quantization.py:27-73)."""
    if axis not in (0, -1):
        raise ValueError("axis parameter must be 0 (first axis) or -1 (last axis)")
    if qtype.bits == 8:
        if shift is not None:
            raise ValueError("shift cannot be specified for 8-bit qtypes")
        if group_size is not None:
            raise ValueError("group_size cannot be specified for 8-bit qtypes.")
        if t.shape[axis] == 1:
            axis = None  # a single feature along the axis is per-tensor quantization
        return WeightQBytesTensor.quantize(t, qtype, axis, scale, activation_qtype, optimized)
    if shift is None:
        raise ValueError("shift must be specified for qtypes lower than 8-bit")
    return WeightQBitsTensor.quantize(t, qtype, axis, group_size, scale, shift, optimized)
