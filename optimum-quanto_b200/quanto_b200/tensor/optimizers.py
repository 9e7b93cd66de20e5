"""Scale / shift search used when a float weight is quantized (offline; not on the hot path).

AbsmaxOptimizer: optimum/quanto/tensor/optimizers/absmax_optimizer.py:26-36
MaxOptimizer   : optimum/quanto/tensor/optimizers/max_optimizer.py:26-37 + affine_optimizer.py:27-64
HqqOptimizer   : optimum/quanto/tensor/optimizers/hqq_optimizer.py:28-87
"""
from typing import Optional, Tuple

import torch

from .grouped import group
from .qtype import qint2, qint4, qtype

__all__ = ["Optimizer", "SymmetricOptimizer", "AffineOptimizer", "AbsmaxOptimizer", "MaxOptimizer", "HqqOptimizer"]


class Optimizer:
    def __call__(self, base, qtype, axis, group_size=None):
        raise NotImplementedError


class SymmetricOptimizer(Optimizer):
    def __call__(self, base: torch.Tensor, qtype: qtype, axis: Optional[int] = None) -> torch.Tensor:
        if axis not in (None, 0, -1):
            raise ValueError("axis parameter must be None, 0 (first axis) or -1 (last axis)")
        if axis is not None and base.shape[axis] == 1:
            axis = None
        scale = self.optimize(base, qtype, axis)
        assert scale.dtype == base.dtype
        return scale

    def optimize(self, base, qtype, axis):
        raise NotImplementedError


class AbsmaxOptimizer(SymmetricOptimizer):
    def optimize(self, base, qtype, axis=None):
        mag = base.abs()
        if axis is None:
            top = mag.max()
        else:
            dims = list(range(1, base.ndim)) if axis == 0 else list(range(base.ndim - 1))
            top = mag.amax(dim=dims, keepdim=True)
        return top / qtype.qmax


class AffineOptimizer(Optimizer):
    def __call__(self, base, qtype, axis, group_size=None, zeropoint=False) -> Tuple[torch.Tensor, torch.Tensor]:
        if axis not in (0, -1):
            raise ValueError("axis parameter must be 0 (first axis) or -1 (last axis)")
        if group_size is not None:
            base = group(base, axis, group_size)
        if base.shape[axis] == 1:
            axis = None
        scale, shift = self.optimize(base, qtype, axis)
        assert scale.dtype == base.dtype and shift.dtype == base.dtype
        if zeropoint:
            shift = torch.clamp(torch.round(shift / scale), 0, 2**qtype.bits - 1).to(torch.uint8)
        return scale, shift

    def optimize(self, base, qtype, axis):
        raise NotImplementedError


class MaxOptimizer(AffineOptimizer):
    def optimize(self, base, qtype, axis):
        dims = list(range(1, base.ndim)) if axis == 0 else list(range(base.ndim - 1))
        lo = base.amin(dim=dims, keepdim=True)
        hi = base.amax(dim=dims, keepdim=True)
        levels = 2**qtype.bits - 1
        return (hi - lo) / levels, -lo


def shrink_lp_op(x: torch.Tensor, beta: float, lp_norm: float) -> torch.Tensor:
    """The shrinking operator of HQQ (hqq_optimizer.py:28-34)."""
    if lp_norm == 1:
        return torch.sign(x) * torch.nn.functional.relu(torch.abs(x) - 1.0 / beta)
    return torch.sign(x) * torch.nn.functional.relu(torch.abs(x) - (1.0 / beta) * torch.pow(torch.abs(x), lp_norm - 1))


class HqqOptimizer(MaxOptimizer):
    """Half-Quadratic Quantization shift search ("Half-Quadratic Quantization of Large Machine Learning Models",
    Badri and Shaji): starting from MaxOptimizer's scale and shift, refine the shift by alternating an lp shrink of
    the quantization error with a per-group mean, while the mean absolute error keeps falling.

    A CUDA bf16 / fp16 weight quantized along axis 0 to qint4 / qint2 runs the fused quanto::quantize_qbits_hqq op
    (two launches, no host synchronisation unless `verbose`); everything else, and whatever the op declines, runs the
    torch composition in `optimize`, on any device.
    """

    def __init__(self, lp_norm: Optional[float] = 0.7, beta: Optional[int] = 1e1, kappa: Optional[float] = 1.01,
                 iters: Optional[int] = 20, verbose: Optional[bool] = False) -> None:
        self.lp_norm = lp_norm
        self.beta = beta
        self.kappa = kappa
        self.iters = iters
        self.verbose = verbose

    def __call__(self, base, qtype, axis, group_size=None, zeropoint=False) -> Tuple[torch.Tensor, torch.Tensor]:
        fused = self.fused(base, qtype, axis, group_size, zeropoint)
        if fused is not None:
            return fused[1], fused[2]
        return super().__call__(base, qtype, axis, group_size, zeropoint)

    def fused(self, base, qtype, axis, group_size=None, zeropoint=False):
        """(packed, scale, shift) from quanto::quantize_qbits_hqq, or None where the composition has to run."""
        group = group_size or (base.shape[1] if base.ndim == 2 else 0)
        if (axis != 0 or not base.is_cuda or base.ndim != 2 or base.dtype not in (torch.float16, torch.bfloat16)
                or qtype not in (qint2, qint4) or group <= 0 or base.shape[1] % group != 0
                or base.numel() // group < 2):  # a single group is quantized along no axis (affine_optimizer.py:54)
            return None
        from .. import _native

        try:
            packed, scale, shift, errors = torch.ops.quanto.quantize_qbits_hqq(
                base.detach(), qtype.bits, group, zeropoint, float(self.lp_norm), float(self.beta), float(self.kappa),
                int(self.iters))
        except _native.UnsupportedConfiguration:
            return None
        if self.verbose:
            self.report(errors)
        return packed, scale, shift

    def report(self, errors: torch.Tensor):
        """Print what the reference prints (hqq_optimizer.py:69-80) from the op's `errors`."""
        errors = errors.tolist()
        if self.iters == 0:
            return
        accepted = int(errors[self.iters + 1])
        print(f"Start error: {errors[0]:.6f}")
        for i in range(min(accepted + 1, self.iters)):
            print(f"HQQ error at it #{i}: {errors[i + 1]:.6f}")

    def optimize(self, base: torch.Tensor, qtype: qtype, axis: Optional[int]):
        scale, shift = super().optimize(base, qtype, axis)
        levels = 2**qtype.bits - 1
        best_error = None
        beta = self.beta
        data = torch.clamp(torch.round((base + shift) / scale), 0, levels).to(torch.uint8)  # quantize_affine
        for i in range(self.iters):
            error = base - (scale * data - shift)
            if best_error is None:
                best_error = float(torch.abs(error).mean())
                if self.verbose:
                    print(f"Start error: {best_error:.6f}")
            e = shrink_lp_op(error, beta, self.lp_norm)
            mean_axis = 0 if axis == -1 else -1
            hqq_shift = torch.mean(data * scale - (base - e), axis=mean_axis, keepdim=True)
            data = torch.clamp(torch.round((base + hqq_shift) / scale), 0, levels).to(torch.uint8)
            mean_error = float(torch.abs(base - (scale * data - hqq_shift)).mean())
            if self.verbose:
                print(f"HQQ error at it #{i}: {mean_error:.6f}")
            if mean_error < best_error:
                best_error = mean_error
                shift = hqq_shift
                beta *= self.kappa
            else:
                break
        return scale, shift
