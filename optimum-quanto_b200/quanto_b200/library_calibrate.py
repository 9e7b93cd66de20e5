"""`quanto::absmax_update_`: one calibration step of a per-tensor activation scale, in place, as one launch.

The reference's Calibration (optimum/quanto/calibrate.py:31-34, 37-61) evaluates `absmax_scale` and then
`_updated_scale`, about seven ATen launches and a host synchronisation (`torch.all(scale == 1)` read as a Python bool)
per scale, and rebinds the module's buffer to the result.  This op reads the activation once and updates the 0-d
`scale` buffer where it is: the `scale == 1` test is made on the device, so nothing waits for the host and a CUDA graph
can capture and replay a calibration step.

Defined here rather than in library.py so that each module registers and fakes exactly the ops it defines.
"""
import torch

from . import _native as N
from .library import _FLOATS, _bind_cuda, _define, _lib

__all__ = []

_define("absmax_update_", "(Tensor(a!) scale, Tensor base, float qmax, float momentum) -> ()")


def _check_absmax_update(scale, base, qmax):
    """The argument checks of quanto::absmax_update_ (the CUDA implementation and the fake)."""
    if base.dtype not in _FLOATS:
        raise ValueError(f"absmax_update_: the tensor must be float32, float16 or bfloat16 (got {base.dtype})")
    if base.numel() == 0:
        raise ValueError("absmax_update_: the tensor is empty")
    if scale.dtype != base.dtype:
        raise ValueError(f"absmax_update_: the scale is {scale.dtype}, the tensor {base.dtype}")
    if scale.numel() != 1:
        raise ValueError(f"absmax_update_: the scale must be one element (got shape {list(scale.shape)})")
    if scale.device != base.device:
        raise ValueError(f"absmax_update_: the scale is on {scale.device}, the tensor on {base.device}")
    if not qmax > 0:
        raise ValueError(f"absmax_update_: qmax must be positive (got {qmax})")


def absmax_update_cuda(scale, base, qmax, momentum):
    """scale = new if scale == 1 else momentum * scale + new * (1 - momentum), new = max|base| / qmax, in place."""
    _check_absmax_update(scale, base, qmax)
    base = base.contiguous()
    scratch = torch.empty(2, dtype=torch.int32, device=base.device)
    with torch.cuda.device(base.device):
        lib = N.load()
        N.check(lib.qb200_absmax_update(N.ptr(base), N.ptr(scale), N.ptr(scratch), base.numel(),
                                        N.DTYPE_CODE[base.dtype], float(qmax), float(momentum),
                                        N.stream_ptr(base.device)), "quanto::absmax_update_")


_bind_cuda("absmax_update_", absmax_update_cuda)


def _absmax_update_fake(scale, base, qmax, momentum):
    _check_absmax_update(scale, base, qmax)


FAKE_IMPLS = {"absmax_update_": _absmax_update_fake}
for _name, _fake in FAKE_IMPLS.items():
    torch.library.register_fake("quanto::" + _name, _fake, lib=_lib)
