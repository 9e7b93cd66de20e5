"""Quantized `torch.nn.Linear`, `torch.nn.Conv2d` and `torch.nn.LayerNorm` (the callers of the hot path).

`QLinear.forward` is `F.linear(input, self.qweight, bias)` exactly as optimum/quanto/nn/qlinear.py:49-50; the
weight's `__torch_function__` turns that into one `quanto::qbytes_mm` or `quanto::qbits_mm` launch.  `QConv2d.forward`
is `self._conv_forward(input, self.qweight, self.bias)` as optimum/quanto/nn/qconv2d.py; F.conv2d on a frozen weight
becomes one `quanto::qbits_conv2d` / `quanto::qbytes_conv2d` launch where the kernel takes the problem.
`QLayerNorm` (optimum/quanto/nn/qlayernorm.py) runs F.layer_norm and its output quantisation as one
`quanto::qbytes_layer_norm` launch when no gradient is needed (library_norm.qlayernorm_forward).
`QModuleMixin` keeps the reference's constructor arguments, hooks, state-dict keys and freeze semantics
(optimum/quanto/nn/qmodule.py:94-312).
"""
from typing import Optional, Union

import torch

from . import _native
from .calibrate import calibrating
from .library_norm import qlayernorm_forward
from .tensor import (AbsmaxOptimizer, ActivationQBytesTensor, HqqOptimizer, MaxOptimizer, Optimizer, QTensor,
                     SymmetricOptimizer, PackedTensor, WeightQBitsTensor, WeightQBytesTensor, qint2, qint4, qtype, qtypes,
                     quantize_activation, quantize_weight)

__all__ = ["QModuleMixin", "QLinear", "QConv2d", "QLayerNorm", "freeze"]


def _pick_group_size(in_features: int) -> Optional[int]:
    """128, stepping down by 32 until it divides in_features (nn/qmodule.py:121-129); None = per-axis."""
    g = 128
    if in_features <= g:
        return None
    while in_features % g != 0 and g > 32:
        g -= 32
    return g if in_features % g == 0 else None


class QModuleMixin:
    def __init__(self, *args, weights: Optional[Union[qtype, str]] = None,
                 activations: Optional[Union[qtype, str]] = None, optimizer: Optional[Optimizer] = None,
                 quantize_input: Optional[bool] = False, device: Optional[torch.device] = None, **kwargs):
        mro = self.__class__.__mro__
        if torch.nn.Module not in mro:
            raise TypeError("Quantized modules must inherit from a torch.nn.Module class")
        if mro.index(__class__) > mro.index(torch.nn.Module):
            raise TypeError(
                "QModuleMixin must be placed before any torch.nn.Module class in quantized module inheritance."
            )
        super().__init__(*args, device=device, **kwargs)
        if weights is not None and not isinstance(weights, qtype):
            weights = qtypes[weights]
        if activations is not None and not isinstance(activations, qtype):
            activations = qtypes[activations]
        self.weight_qtype = weights
        self.weight_group_size = None
        if self.weight_qtype in (qint2, qint4):
            out_features = self.weight.shape[0]
            self.weight_group_size = _pick_group_size(self.weight.numel() // out_features)
        self.activation_qtype = activations
        self._quantize_hooks = {}
        if activations is not None:
            if quantize_input:
                self._quantize_hooks["input"] = self.register_forward_pre_hook(self.quantize_input)
            self._quantize_hooks["output"] = self.register_forward_hook(self.quantize_output)
        if optimizer is None and self.weight_qtype is not None:
            optimizer = AbsmaxOptimizer() if self.weight_qtype.bits == 8 else MaxOptimizer()
        self.optimizer = optimizer
        scale_dtype = torch.float32 if self.weight is None else self.weight.dtype
        self.register_buffer("input_scale", torch.ones((), dtype=scale_dtype, device=device))
        self.register_buffer("output_scale", torch.ones((), dtype=scale_dtype, device=device))

    def disable_output_quantization(self):
        if "output" in self._quantize_hooks:
            self._quantize_hooks.pop("output").remove()

    # ------------------------------------------------------------------ (de)serialization: canonical packing only
    def _save_to_state_dict(self, destination, prefix, keep_vars):
        if self.weight_qtype is None or not self.frozen:
            destination[prefix + "weight"] = self.weight if (self.weight is None or keep_vars) else self.weight.detach()
        else:
            self.weight.save_to_state_dict(destination, prefix + "weight.", keep_vars)
        if self.bias is not None:
            destination[prefix + "bias"] = self.bias if keep_vars else self.bias.detach()
        destination[prefix + "input_scale"] = self.input_scale if keep_vars else self.input_scale.detach()
        destination[prefix + "output_scale"] = self.output_scale if keep_vars else self.output_scale.detach()

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                              error_msgs):
        weight_name = prefix + "weight"
        if self.weight_qtype is not None and weight_name not in state_dict:
            weight_prefix = weight_name + "."
            if self.weight_qtype.bits == 8:
                w = WeightQBytesTensor.load_from_state_dict(
                    state_dict, weight_prefix, qtype=self.weight_qtype, axis=0, size=self.weight.size(),
                    stride=self.weight.stride(), activation_qtype=self.activation_qtype, missing_keys=missing_keys)
            else:
                w = WeightQBitsTensor.load_from_state_dict(
                    state_dict, weight_prefix, qtype=self.weight_qtype, axis=0, group_size=self.weight_group_size,
                    size=self.weight.size(), stride=self.weight.stride(), missing_keys=missing_keys)
            if w is not None:
                w = w.optimize()
                if local_metadata.get("assign_to_params_buffers", False):
                    self.weight = torch.nn.Parameter(w, requires_grad=False)
                else:
                    self.weight = torch.nn.Parameter(w.to(self.weight.device), requires_grad=False)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, False, missing_keys, unexpected_keys,
                                      error_msgs)

    # ------------------------------------------------------------------------------------------ construction
    @classmethod
    def from_module(cls, module: torch.nn.Module, weights: Optional[qtype] = None,
                    activations: Optional[qtype] = None, optimizer: Optional[Optimizer] = None):
        qmodule = cls.qcreate(module, weights, activations, optimizer, device="meta")
        if qmodule is None:
            return None
        device = torch.device("cpu") if module.weight is None else module.weight.device
        qmodule = qmodule.to_empty(device=device)
        qmodule.input_scale = torch.ones_like(qmodule.input_scale)
        qmodule.output_scale = torch.ones_like(qmodule.output_scale)
        with torch.no_grad():
            qmodule.weight = module.weight
            if module.bias is not None:
                qmodule.bias = module.bias
        return qmodule.to(device)

    @classmethod
    def qcreate(cls, module, weights, activations=None, optimizer=None, device=None):
        raise NotImplementedError

    # ---------------------------------------------------------------------------------------------- forward
    @property
    def qweight(self):
        if self.weight_qtype is None:
            return None
        if isinstance(self.weight, QTensor):
            return self.weight  # frozen
        fused = self._fused_qweight()
        if fused is not None:
            return fused
        if isinstance(self.optimizer, SymmetricOptimizer):
            scale = self.optimizer(self.weight, qtype=self.weight_qtype, axis=0)
            shift = None
        else:
            scale, shift = self.optimizer(self.weight, qtype=self.weight_qtype, axis=0,
                                          group_size=self.weight_group_size)
        return quantize_weight(self.weight, qtype=self.weight_qtype, axis=0, scale=scale, shift=shift,
                               group_size=self.weight_group_size, activation_qtype=self.activation_qtype)

    def _fused_qweight(self):
        """Range search + quantisation (+ packing) of a CUDA weight as ONE launch (SURVEY 8f rank 1).

        Taken when the result cannot need a gradient (freeze(), inference with dynamic weights) and the optimizer is
        exactly the default one, so the result equals `optimizer(...)` + `quantize_weight(...)` of the reference's
        CPU path bit for bit (nn/qmodule.py:245-266 with max_optimizer.py:26-37 / absmax_optimizer.py:29-36).
        Returns None when the composition of separate ops has to run instead.

        A conv weight [Cout, Cin, kh, kw] is quantized as the linear weight [Cout, Cin * kh * kw] it flattens to (the
        reference groups the row-major flattening, tensor/grouped.py); only the per-axis tensors are then given back the
        4-D shapes the composition produces (packed [ceil(Cout / 2), Cin, kh, kw], scale / shift [Cout, 1, 1, 1]).
        """
        w = self.weight
        if (w is None or not w.is_cuda or w.ndim not in (2, 4)
                or w.dtype not in (torch.float32, torch.float16, torch.bfloat16)
                or (torch.is_grad_enabled() and w.requires_grad)):
            return None
        w2 = w.detach().reshape(w.shape[0], -1)
        coef_shape = (w.shape[0],) + (1,) * (w.ndim - 1)  # per-axis scales / shifts, as the optimizers keep them
        qt = self.weight_qtype

        def qbits(packed, scale, shift):
            group = self.weight_group_size or w2.shape[1]
            rows = w.numel() // group
            if self.weight_group_size is None and w.ndim == 4:
                data = PackedTensor(packed.reshape((packed.shape[0],) + tuple(w.shape[1:])), qt.bits, w.size(),
                                    w.stride())
                scale, shift = scale.reshape(coef_shape), shift.reshape(coef_shape)
            else:
                data = PackedTensor(packed, qt.bits, torch.Size([rows, group]), (group, 1))
            return WeightQBitsTensor(qt, 0, self.weight_group_size, w.size(), w.stride(), data, scale, shift)

        if qt in (qint2, qint4) and type(self.optimizer) is MaxOptimizer:
            group = self.weight_group_size or w2.shape[1]
            try:
                packed, scale, shift = torch.ops.quanto.quantize_qbits_max(w2, qt.bits, group, False)
            except _native.UnsupportedConfiguration:
                return None
            return qbits(packed, scale, shift)
        if qt in (qint2, qint4) and type(self.optimizer) is HqqOptimizer:
            if w.ndim == 4 and self.weight_group_size is None:
                # per-axis HQQ reduces a whole [Cin, kh, kw] slice: the reference's float sums over the 4-D tensor run
                # in another order than over the [Cout, K] rows the kernel reproduces, so its shifts may differ
                return None
            group = self.weight_group_size or w2.shape[1]
            fused = self.optimizer.fused(w2, qt, 0, group)
            if fused is None:
                return None
            return qbits(*fused)
        if (qt is not None and qt.bits == 8 and type(self.optimizer) is AbsmaxOptimizer and w.shape[0] > 1
                and qt.dtype in (torch.int8, torch.float8_e4m3fn, torch.float8_e5m2)):
            data, scale = torch.ops.quanto.quantize_qbytes_absmax(w2, qt.dtype)
            return WeightQBytesTensor(qt, 0, w.size(), w.stride(), data.reshape(w.shape), scale.reshape(coef_shape),
                                      self.activation_qtype)
        return None

    def quantize_input(self, module, input):
        input = input[0]
        if isinstance(input, ActivationQBytesTensor):
            # compared by storage dtype (one per 8-bit qtype): under torch.compile an activation created inside the
            # graph exposes only tensors and literals, not its qtype object
            if input._data.dtype != self.activation_qtype.dtype:
                raise ValueError(
                    "Models with heterogeneous quantized activations are not supported:"
                    f" expected {self.activation_qtype.name} input but got {input.qtype.name} instead."
                )
            return input
        return quantize_activation(input, qtype=self.activation_qtype, scale=self.input_scale)

    def quantize_output(self, module, input, output):
        if isinstance(output, ActivationQBytesTensor) and output._data.dtype == self.activation_qtype.dtype:
            return output  # QLinear.forward already quantised it in the GEMM epilogue (one launch, see below)
        return quantize_activation(output, qtype=self.activation_qtype, scale=self.output_scale)

    def freeze(self):
        with torch.no_grad():  # the frozen weight never carries a graph; lets CUDA weights take the one-launch path
            qweight = self.qweight
        if qweight is not None:
            self.weight = torch.nn.Parameter(qweight, requires_grad=False)

    @property
    def frozen(self):
        return isinstance(self.weight, QTensor)


class QLinear(QModuleMixin, torch.nn.Linear):
    @classmethod
    def qcreate(cls, module, weights: qtype, activations: Optional[qtype] = None,
                optimizer: Optional[Optimizer] = None, device: Optional[torch.device] = None):
        return cls(module.in_features, module.out_features, module.bias is not None, dtype=module.weight.dtype,
                   device=device, weights=weights, activations=activations, optimizer=optimizer, quantize_input=True)

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        fused = self._forward_quantized_output(input)
        if fused is not None:
            return fused
        return torch.nn.functional.linear(input, self.qweight, bias=self.bias)

    def _forward_quantized_output(self, input):
        """Quantized activations in AND out with a frozen 8-bit weight: the linear, its bias and the `quantize_output`
        hook (nn/qmodule.py:300-302) as ONE `quanto::qbytes_linear_quantized` launch (SURVEY 8f rank 2) -- the [M, N]
        result is never written in 16 bits and read back.  Bit-identical to `F.linear` followed by the hook; inference
        only (no graph).  Returns None when the ordinary path has to run, and while a `Calibration` mode needs to
        see the float output."""
        w = self.weight
        if ("output" not in self._quantize_hooks or not isinstance(input, ActivationQBytesTensor)
                or not isinstance(w, WeightQBytesTensor) or not w._data.is_cuda or w.axis != 0 or w.ndim != 2
                or input._data.dtype != self.activation_qtype.dtype
                or (torch.is_grad_enabled() and (input.requires_grad or w.requires_grad)) or calibrating()):
            return None
        scales = input._scale * w._scale  # in the module dtype, one rounding (tensor/weights/qbytes.py:72-73)
        data = torch.ops.quanto.qbytes_linear_quantized(input._data, w._data, scales, self.bias, self.output_scale,
                                                        self.activation_qtype.dtype)
        return ActivationQBytesTensor(self.activation_qtype, data.size(), data.stride(), data, self.output_scale)


class QConv2d(QModuleMixin, torch.nn.Conv2d):
    """optimum/quanto/nn/qconv2d.py: the weight is quantized along axis 0 with the group size of its flattening
    Cin * kh * kw; the input is not quantized (quantize_input stays False), the output is when `activations` is set."""

    @classmethod
    def qcreate(cls, module, weights: qtype, activations: Optional[qtype] = None,
                optimizer: Optional[Optimizer] = None, device: Optional[torch.device] = None):
        return cls(in_channels=module.in_channels, out_channels=module.out_channels, kernel_size=module.kernel_size,
                   stride=module.stride, padding=module.padding, dilation=module.dilation, groups=module.groups,
                   bias=module.bias is not None, padding_mode=module.padding_mode, dtype=module.weight.dtype,
                   device=device, weights=weights, activations=activations, optimizer=optimizer)

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        # a padding_mode other than 'zeros' pads with F.pad here, then the conv itself runs with padding 0
        return self._conv_forward(input, self.qweight, self.bias)


class QLayerNorm(QModuleMixin, torch.nn.LayerNorm):
    """optimum/quanto/nn/qlayernorm.py: created only with `activations` set; the weight and bias are never quantized and
    the output is quantized per tensor with `output_scale`."""

    @classmethod
    def qcreate(cls, module, weights: Optional[qtype] = None, activations: Optional[qtype] = None,
                optimizer: Optional[Optimizer] = None, device: Optional[torch.device] = None):
        if activations is None:
            return None
        dtype = None if module.weight is None else module.weight.dtype
        return cls(module.normalized_shape, module.eps, module.elementwise_affine, module.bias is not None, dtype=dtype,
                   device=device, weights=None, activations=activations, optimizer=None)

    def forward(self, input: torch.Tensor) -> torch.Tensor:
        if not calibrating():  # the output calibration has to see F.layer_norm's float output
            out = qlayernorm_forward(self, input, ActivationQBytesTensor, "output" in self._quantize_hooks)
            if out is not None:
                return out
        return torch.nn.functional.layer_norm(input, self.normalized_shape, self.weight, self.bias, self.eps)


def freeze(model: torch.nn.Module):
    """Freeze every quantized module of `model` (optimum/quanto/quantize.py:142-146)."""
    for m in model.modules():
        if isinstance(m, QModuleMixin):
            m.freeze()
