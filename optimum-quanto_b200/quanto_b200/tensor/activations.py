"""Per-tensor 8-bit quantized activations (optimum/quanto/tensor/activations/qbytes.py:28-92, quantization.py:24-39).

Construction through `quanto::quantize_symmetric` (one sm_90a kernel), flatten/unflatten, and the reference's aten op
table (qbytes_ops.py, ported in activation_ops.py): layout ops keep the tensor quantized, `bmm` of two qint8 activations
and `_softmax` run on the library's kernels, every other op dequantizes.  `F.linear` never reaches the table because the
weight's `__torch_function__` intercepts first.
"""
import ast

import torch
from torch.autograd import Function

from .qtensor import QBytesTensor, qfallback
from .qtype import qtype, qtypes

__all__ = ["ActivationQBytesTensor", "quantize_activation"]


class ActivationQBytesQuantizer(Function):
    @staticmethod
    def forward(ctx, base, qtype, scale):
        if qtype.bits != 8:
            raise ValueError("QBytesTensor can only be of 8-bit qtype")
        data = torch.ops.quanto.quantize_symmetric(base, dtype=qtype.dtype, axis=None, scale=scale)
        return ActivationQBytesTensor(qtype, base.size(), base.stride(), data, scale)

    @staticmethod
    def backward(ctx, gO):
        return gO, None, None, None, None, None


class ActivationQBytesTensor(QBytesTensor):
    @staticmethod
    def __new__(cls, qtype, size, stride, data, scale, requires_grad=False):
        assert data.device == scale.device
        return torch.Tensor._make_wrapper_subclass(
            cls, size, strides=stride, dtype=scale.dtype, device=data.device, requires_grad=requires_grad
        )

    def __init__(self, qtype, size, stride, data, scale, requires_grad=False):
        super().__init__(qtype, None, size, stride, data, scale, requires_grad)

    @classmethod
    def quantize(cls, base, qtype, scale):
        return ActivationQBytesQuantizer.apply(base, qtype, scale)

    def __tensor_flatten__(self):
        meta = {"qtype": self._qtype.name, "size": str(list(self.size())), "stride": str(list(self.stride()))}
        return ["_data", "_scale"], meta

    @staticmethod
    def __tensor_unflatten__(inner_tensors, meta, outer_size, outer_stride):
        assert len(inner_tensors) == 2 and len(meta) == 3
        # under tracing the outer size may be symbolic (a dynamic token count): it is passed in, not parsed from meta
        size = ast.literal_eval(meta["size"]) if outer_size is None else outer_size
        stride = ast.literal_eval(meta["stride"]) if outer_stride is None else outer_stride
        return ActivationQBytesTensor(
            qtypes[meta["qtype"]],
            size,
            stride,
            inner_tensors["_data"],
            inner_tensors["_scale"],
        )

    @classmethod
    def __torch_dispatch__(cls, op, types, args, kwargs=None):
        kwargs = dict(kwargs or {})
        packet = op.overloadpacket
        qdispatch = activation_ops.get_qbytestensor_op_dispatch(packet)
        if qdispatch is not None:
            return qdispatch(*args, **kwargs)
        return qfallback(packet, *args, **kwargs)


def quantize_activation(t: torch.Tensor, qtype: qtype, scale: torch.Tensor):
    if scale.numel() != 1:
        raise ValueError("Parameter scale must be a scalar because activations can only be quantized per-tensor")
    return ActivationQBytesTensor.quantize(t, qtype, scale)


from . import activation_ops  # noqa: E402  (the op table refers to the class above)
