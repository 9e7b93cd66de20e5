"""Model-level API: quantize, freeze, quantization_map and requantize (optimum/quanto/quantize.py, nn/qmodule.py).

The usual flow is `quantize(model, weights=qint8, activations=qint8)`, then `with Calibration(): model(samples)` to set
the activation scales, then `freeze(model)`.  The frozen model's `state_dict()` carries the packed weights and both
scales; `requantize(fresh_model, state_dict, quantization_map(model))` rebuilds the quantized modules and loads it.
"""
from fnmatch import fnmatch
from typing import Any, Dict, List, Optional, Union

import torch

from .nn import QConv2d, QLayerNorm, QLinear, QModuleMixin, freeze
from .tensor import Optimizer, qtype

__all__ = ["quantize_module", "quantize", "freeze", "requantize", "quantization_map"]

# float module class -> its quantized counterpart, tried in this order
_QMODULES = ((torch.nn.Linear, QLinear), (torch.nn.Conv2d, QConv2d), (torch.nn.LayerNorm, QLayerNorm))


def quantize_module(module: torch.nn.Module, weights: Optional[Union[qtype, str]] = None,
                    activations: Optional[Union[qtype, str]] = None, optimizer: Optional[Optimizer] = None):
    """The quantized counterpart of `module`, or None when it has none (a LayerNorm has one only with activations)."""
    for cls, qcls in _QMODULES:
        if isinstance(module, cls):
            return qcls.from_module(module, weights=weights, activations=activations, optimizer=optimizer)
    return None


def _set_module_by_name(model: torch.nn.Module, name: str, child: torch.nn.Module):
    parent_name, _, attr = name.rpartition(".")
    setattr(model.get_submodule(parent_name) if parent_name else model, attr, child)


def _quantize_submodule(model, name, module, weights=None, activations=None, optimizer=None):
    qmodule = quantize_module(module, weights=weights, activations=activations, optimizer=optimizer)
    if qmodule is not None:
        _set_module_by_name(model, name, qmodule)
        qmodule.name = name
        # the quantized module holds the tensors now: drop the original's references to them
        for pname, _ in list(module.named_parameters()):
            setattr(module, pname, None)


def quantize(model: torch.nn.Module, weights: Optional[Union[str, qtype]] = None,
             activations: Optional[Union[str, qtype]] = None, optimizer: Optional[Optimizer] = None,
             include: Optional[Union[str, List[str]]] = None, exclude: Optional[Union[str, List[str]]] = None):
    """Replace, in place, every submodule of `model` that has a quantized counterpart.

    `include` / `exclude` are fnmatch patterns (not regular expressions) on the submodule names: a module is quantized
    only when its name matches one of the include patterns (if given) and none of the exclude patterns (if given).
    """
    if isinstance(include, str):
        include = [include]
    if isinstance(exclude, str):
        exclude = [exclude]
    for name, m in model.named_modules():
        if include is not None and not any(fnmatch(name, p) for p in include):
            continue
        if exclude is not None and any(fnmatch(name, p) for p in exclude):
            continue
        _quantize_submodule(model, name, m, weights=weights, activations=activations, optimizer=optimizer)


def _qtype_name(t: Optional[qtype]) -> str:
    return "none" if t is None else t.name


def _qtype_or_none(name: str) -> Optional[str]:
    return None if name == "none" else name


def quantization_map(model: torch.nn.Module) -> Dict[str, Dict[str, str]]:
    """{submodule name: {"weights": qtype name or "none", "activations": qtype name or "none"}} of every quantized
    submodule: what `requantize` needs besides the state dict."""
    return {name: {"weights": _qtype_name(m.weight_qtype), "activations": _qtype_name(m.activation_qtype)}
            for name, m in model.named_modules() if isinstance(m, QModuleMixin)}


def _on_cpu(t: torch.Tensor) -> torch.Tensor:
    """`t` on the CPU; a meta tensor becomes uninitialised CPU storage of its shape, for load_state_dict to fill."""
    return torch.empty_like(t, device="cpu") if t.is_meta else t.cpu()


def requantize(model: torch.nn.Module, state_dict: Dict[str, Any], quantization_map: Dict[str, Dict[str, str]],
               device: Optional[torch.device] = None):
    """Quantize `model` (on any device, meta included) as `quantization_map` says and load `state_dict` into it.

    The quantized modules are built, every parameter and buffer is materialised on the CPU and then moved to `device`
    (default: the device of the model's first parameter, or the CPU for a meta model), and the state dict is loaded
    with strict=False: the quantized modules' `_load_from_state_dict` turns the serialized weight tensors back into
    frozen QTensor weights.
    """
    if device is None:
        first = next(model.parameters()).device
        device = torch.device("cpu") if first.type == "meta" else first
    targets = [(name, m, quantization_map[name]) for name, m in model.named_modules() if name in quantization_map]
    for name, m, qconfig in targets:
        _quantize_submodule(model, name, m, weights=_qtype_or_none(qconfig["weights"]),
                            activations=_qtype_or_none(qconfig["activations"]))
    for m in model.modules():
        for key, p in m._parameters.items():
            if p is not None:
                m._parameters[key] = torch.nn.Parameter(_on_cpu(p), requires_grad=p.requires_grad)
        for key, b in m._buffers.items():
            if b is not None:
                m._buffers[key] = _on_cpu(b)
    model.to(device)
    model.load_state_dict(state_dict, strict=False)
