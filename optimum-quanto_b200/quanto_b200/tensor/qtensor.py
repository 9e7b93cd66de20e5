"""The QTensor data model: base class, the dequantising fallback, and the two storage classes (8-bit values with a scale;
sub-byte packed values with a per-group scale and shift).  Interface of optimum/quanto/tensor/qtensor.py:21-85,
tensor/qbytes.py:23-50 and tensor/qbits.py:27-68 in one module."""
import torch
from torch.utils import _pytree as pytree

__all__ = ["QTensor", "qfallback", "QBytesTensor", "QBitsTensor"]


def qfallback(fn, *args, **kwargs):
    """Run `fn` on dequantised copies of every QTensor argument (used for ops without a quantized kernel)."""
    args, kwargs = pytree.tree_map_only(QTensor, lambda q: q.dequantize(), (args, kwargs or {}))
    return fn(*args, **kwargs)


class QTensor(torch.Tensor):
    def __init__(self, qtype, axis):
        self._qtype = qtype
        self._axis = axis

    def dequantize(self):
        raise NotImplementedError

    @property
    def axis(self):
        return self._axis

    @property
    def qtype(self):
        return self._qtype

    def numpy(self):
        return self.dequantize().cpu().numpy()

    def save_to_state_dict(self, destination, prefix, keep_vars):
        """Flatten into plain tensors: `<prefix>_data`, `<prefix>_scale`, ... (nested subclasses recurse)."""

        def flatten(t, pfx):
            names, _ = t.__tensor_flatten__()
            for name in names:
                inner = getattr(t, name)
                if type(inner) is torch.Tensor:
                    destination[pfx + name] = inner if keep_vars else inner.detach()
                else:
                    flatten(inner, pfx + name + ".")

        flatten(self, prefix)

    def equal(self, other):
        if type(self) is not type(other):
            return False
        names, meta = self.__tensor_flatten__()
        _, other_meta = other.__tensor_flatten__()
        if any(other_meta[k] != v for k, v in meta.items()):
            return False
        for name in names:
            a, b = getattr(self, name), getattr(other, name)
            if hasattr(a, "_bits") and hasattr(b, "_bits"):  # PackedTensor: compare the packed bytes themselves
                if a._bits != b._bits or a.shape != b.shape:
                    return False
                a, b = a._data, b._data
            if a.dtype != b.dtype:
                return False
            if a.dtype in (torch.float8_e4m3fn, torch.float8_e5m2, torch.float8_e4m3fnuz):
                a, b = a.view(torch.uint8), b.view(torch.uint8)  # bit comparison (torch.equal lacks fp8 on CPU)
            if not torch.equal(a, b):
                return False
        return True


# ----------------------------------------------------------------------------------------------------------------------
# The two storage models.  Both dequantise through ONE straight-through autograd function whose forward is the
# storage class's `_dequantize_impl` (the reference keeps a Function per class: tensor/qbytes.py:23-40,
# tensor/qbits.py:27-52); the gradient of a dequantisation is the identity either way.
# ----------------------------------------------------------------------------------------------------------------------
class _StraightThroughDequantize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, qt):
        return qt._dequantize_impl()

    @staticmethod
    def backward(ctx, grad):
        return grad


class QBytesTensor(QTensor):
    """8 bits per value: `_data` (int8 / float8) and `_scale`; value = scale * data  (tensor/qbytes.py:42-50)."""

    def __init__(self, qtype, axis, size, stride, data, scale, requires_grad=False):
        super().__init__(qtype, axis)
        self._data, self._scale = data, scale

    def __repr__(self):
        return f"{type(self).__name__}({self._data}, scale={self._scale}, dtype={self.dtype})"

    def _dequantize_impl(self):
        payload = self._data.to(self._scale.dtype) if self._data.dtype.is_floating_point else self._data  # fp8: no mul
        return self._scale * payload

    def dequantize(self):
        return _StraightThroughDequantize.apply(self)


class QBitsTensor(QTensor):
    """Fewer than 8 bits per value: `_data` (a PackedTensor of group rows), `_scale`, `_shift` per group
    (tensor/qbits.py:54-68).  value = scale * data - shift, or scale * (data - zero_point) for integer shifts."""

    def __init__(self, qtype, axis, group_size, size, stride, data, scale, shift, requires_grad=False):
        super().__init__(qtype, axis)
        self._data, self._scale, self._shift, self._group_size = data, scale, shift, group_size

    def __repr__(self):
        return f"{type(self).__name__}({self._data}, scale={self._scale}, shift={self._shift}, dtype={self.dtype})"

    def _one_launch_dequant_ok(self) -> bool:
        """Canonical axis-0 storage on a CUDA device: `quanto::dequantize_qbits` does the whole chain in one kernel."""
        packed = getattr(self._data, "_data", None)
        return (
            packed is not None and hasattr(self._data, "_bits") and packed.is_cuda
            and self.axis == 0 and len(self.shape) == 2
            and self._group_size is not None and self._group_size % 4 == 0
            and self._scale.dtype in (torch.float32, torch.float16, torch.bfloat16)
            and (not self._shift.dtype.is_floating_point or self._shift.dtype == self._scale.dtype)
        )

    def _dequantize_impl(self):
        if self._one_launch_dequant_ok():
            n, k = self.shape
            return torch.ops.quanto.dequantize_qbits(self._data._data, self._scale, self._shift, n, k,
                                                     self._group_size, self._data._bits)
        # any other layout (axis -1, per-axis, CPU tensors): the reference's chain on ATen ops, same rounding order
        from .grouped import ungroup

        values = self._data.unpack() if hasattr(self._data, "unpack") else self._data
        if self._shift.dtype.is_floating_point:
            out = self._scale * values - self._shift
        else:
            out = self._scale * (values.to(torch.int8) - self._shift.to(torch.int8))  # zero-point leaves first
        return out if self.axis is None else ungroup(out, axis=self.axis, orig_shape=self.shape)

    def dequantize(self):
        return _StraightThroughDequantize.apply(self)
