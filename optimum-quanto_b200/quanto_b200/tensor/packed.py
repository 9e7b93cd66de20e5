"""Sub-byte storage: `pack_weights` and the `PackedTensor` wrapper.

Storage contract (kept bit-for-bit, it is quanto's on-disk format, optimum/quanto/tensor/packed.py:24-163):
rows are split into 8/bits planes of R = ceil(rows / (8/bits)) rows; byte (i, c) holds plane p at bits [p*bits, (p+1)*bits).
For an int4 [N*K/G, G] weight this means: low nibble = out-features [0, N/2), high nibble = [N/2, N), same k.
`unpack()` goes through `torch.ops.quanto.unpack`, i.e. the sm_90a kernel on CUDA tensors.
"""
import ast

import torch
from torch.utils import _pytree as pytree

__all__ = ["PackedTensor", "pack_weights"]


def pack_weights(intweights: torch.Tensor, bits: int) -> torch.Tensor:
    """Pack `bits`-wide unsigned values (one per uint8) along dim 0 into uint8 (planes stacked in the byte)."""
    if bits not in (2, 4):
        raise ValueError("bits must be 2 or 4")
    if intweights.is_cuda:
        return torch.ops.quanto.pack(intweights.to(torch.uint8), bits)  # one sm_90a launch (csrc/freeze.cu)
    # CPU tensors (building / loading a model on the host): the reference's slice-shift-or loop
    per_byte = 8 // bits
    rows = intweights.shape[0]
    packed_rows = -(-rows // per_byte)
    values = intweights.to(torch.uint8)
    packed = torch.zeros((packed_rows,) + tuple(intweights.shape[1:]), dtype=torch.uint8, device=intweights.device)
    for plane in range(per_byte):
        chunk = values[plane * packed_rows : min((plane + 1) * packed_rows, rows)]
        if chunk.shape[0] > 0:
            packed[: chunk.shape[0]] |= chunk << (bits * plane)
    return packed


class PackedTensor(torch.Tensor):
    """uint8 wrapper subclass remembering the logical (unpacked) size."""

    @staticmethod
    def __new__(cls, data, bits, size, stride, requires_grad=False):
        assert data.dtype == torch.uint8
        assert requires_grad is False
        return torch.Tensor._make_wrapper_subclass(
            cls, size, strides=stride, dtype=torch.uint8, device=data.device, requires_grad=False
        )

    def __init__(self, data, bits, size, stride, requires_grad=False):
        self._bits = bits
        self._data = data

    def __repr__(self):
        return f"PackedTensor({self._data}, bits={self._bits}, public_dtype={self.dtype})"

    @classmethod
    def pack(cls, t: torch.Tensor, bits: int = 4):
        assert bits in (2, 4)
        assert t.dtype in (torch.uint8, torch.int8)
        return PackedTensor(pack_weights(t, bits), bits, t.size(), t.stride())

    def unpack(self) -> torch.Tensor:
        planes = torch.ops.quanto.unpack(self._data, self._bits)
        return planes[: self.shape[0]]  # drop the padding rows of an odd row count

    @property
    def bits(self):
        return self._bits

    @property
    def dtype(self):
        return torch.uint8

    @staticmethod
    def load_from_state_dict(state_dict, prefix, bits, size, stride, missing_keys):
        key = prefix + "_data"
        if key not in state_dict:
            missing_keys.append(key)
            return None
        meta = {"bits": str(bits), "size": str(list(size)), "stride": str(stride)}
        return PackedTensor.__tensor_unflatten__({"_data": state_dict.pop(key)}, meta, None, None)

    def __tensor_flatten__(self):
        meta = {"bits": str(self._bits), "size": str(list(self.size())), "stride": str(self.stride())}
        return ["_data"], meta

    @staticmethod
    def __tensor_unflatten__(inner_tensors, meta, outer_size, outer_stride):
        assert len(inner_tensors) == 1 and len(meta) == 3
        return PackedTensor(
            inner_tensors["_data"],
            ast.literal_eval(meta["bits"]),
            ast.literal_eval(meta["size"]),
            ast.literal_eval(meta["stride"]),
        )

    __torch_function__ = torch._C._disabled_torch_function_impl

    @classmethod
    def __torch_dispatch__(cls, op, types, args, kwargs=None):
        kwargs = kwargs or {}
        packet = op.overloadpacket
        if packet is torch.ops.aten.detach:
            t = args[0]
            return PackedTensor(op(t._data), t._bits, t.size(), t.stride())
        if packet in (torch.ops.aten._to_copy, torch.ops.aten.to):
            t = args[0]
            if kwargs.get("dtype", torch.uint8) != torch.uint8:
                raise ValueError(f"PackedTensor are torch.uint8 only and cannot be moved to {kwargs['dtype']}.")
            return PackedTensor(op(t._data, **kwargs), t._bits, t.size(), t.stride())
        args, kwargs = pytree.tree_map_only(PackedTensor, lambda x: x.unpack(), (args, kwargs))
        return op(*args, **kwargs)

    def numpy(self):
        return self.unpack().cpu().numpy()
