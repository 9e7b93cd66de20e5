"""Activation-scale calibration: `absmax_scale` and the `Calibration` mode (optimum/quanto/calibrate.py).

`Calibration` is a torch-function mode with the reference's constructor, global forward hooks and observable
semantics: inside `with Calibration():` every forward of a quantized module with activations updates its
`input_scale` and `output_scale` from the absmax of the float activation, with a momentum.  On CUDA, when the buffer and
the activation share a dtype, each update is one `quanto::absmax_update_` launch on the buffer in place: no host
synchronisation, and the buffer keeps its identity, so a captured calibration step can be replayed.  Every other case
(CPU tensors, mixed dtypes, a tensor the op declines) runs the reference's composition and rebinds the buffer.
"""
from typing import Optional

import torch
from torch.nn.modules.module import register_module_forward_hook, register_module_forward_pre_hook
from torch.overrides import TorchFunctionMode

from . import _native
from . import library_calibrate  # noqa: F401  (registers quanto::absmax_update_)
from .tensor.activations import ActivationQBytesTensor
from .tensor.core import axis_to_dim, dtype_info
from .tensor.qtype import qint8, qtype

__all__ = ["Calibration", "absmax_scale"]

# Private switch for measurements and tests: run every update as the reference's composition, whose
# torch.all(scale == 1) synchronises with the host.
_FORCE_COMPOSITION = False


def absmax_scale(base: torch.Tensor, qtype: qtype = qint8, axis: Optional[int] = None) -> torch.Tensor:
    """scale = max|base| / dtype_info(qtype.dtype).max, per tensor (axis None) or keeping `axis`.

    Per-tensor on a CUDA tensor the |x| + max pair is one reduction kernel (`quanto::absmax`) instead of two ATen
    passes over the activation.  The division is tensor / tensor so that it is a true IEEE division on every device
    (torch's CUDA kernels turn tensor / python-scalar into a multiplication by the reciprocal, one ulp off the
    reference's CPU result).
    """
    info = dtype_info(qtype.dtype)
    if axis is None:
        if base.is_cuda and base.dtype in (torch.float32, torch.float16, torch.bfloat16):
            qranges = torch.ops.quanto.absmax(base)
        else:
            qranges = torch.max(torch.abs(base))
    else:
        qranges = torch.amax(torch.abs(base), dim=axis_to_dim(base, axis), keepdim=True)
    return qranges / torch.tensor(info.max, dtype=base.dtype, device=base.device)


def _updated_scale(scale: torch.Tensor, new_scale: torch.Tensor, momentum: float) -> torch.Tensor:
    """The reference's momentum update: a scale still exactly 1 (never calibrated, or reset there) takes the new one."""
    if torch.all(scale == 1):
        return new_scale
    return momentum * scale + new_scale * (1.0 - momentum)


_FLOATS = (torch.float32, torch.float16, torch.bfloat16)
_INPUT_MOMENTUM = 0.9  # the reference's input hook never receives the mode's momentum (DESIGN.md, calibration quirks)


def _calibrate_scale(module: torch.nn.Module, name: str, base: torch.Tensor, qtype: qtype, momentum: float):
    """Update the per-tensor scale buffer `name` of `module` from the activation `base`: in place through
    quanto::absmax_update_ where it takes the problem, else the reference's composition, which rebinds the buffer."""
    scale = getattr(module, name)
    native = (not _FORCE_COMPOSITION and type(base) is torch.Tensor and base.is_cuda and base.dtype in _FLOATS
              and scale.dtype == base.dtype and scale.device == base.device and scale.numel() == 1
              and base.numel() > 0)
    if native:
        try:
            torch.ops.quanto.absmax_update_(scale, base.detach(), dtype_info(qtype.dtype).max, momentum)
            return
        except _native.UnsupportedConfiguration:
            pass
    setattr(module, name, _updated_scale(scale, absmax_scale(base, qtype), momentum))


def _adopt_input_scale(module: torch.nn.Module, scale: torch.Tensor):
    """input_scale = `scale` (the largest scale of an already quantized input), into the buffer where it fits."""
    buf = module.input_scale
    if not _FORCE_COMPOSITION and buf.is_cuda and (buf.dtype, buf.device, buf.shape) == (scale.dtype, scale.device,
                                                                                           scale.shape):
        buf.copy_(scale)
    else:
        module.input_scale = scale


_entered = 0  # Calibration modes currently entered


def calibrating() -> bool:
    """True while a `Calibration` mode is entered.

    The paths that quantize a module's output inside its kernel (QLinear's fused qint8 epilogue, QLayerNorm's one-launch
    op) stand aside then: the output calibration has to see the float output before the output hook quantizes it.  A
    plain counter rather than a walk of the mode stack, so that torch.compile traces the module forwards that ask."""
    return _entered > 0


def _is_calibrated(module: torch.nn.Module) -> bool:
    from .nn import QModuleMixin  # nn.py consults calibrating(): imported here to keep the import graph acyclic

    return isinstance(module, QModuleMixin) and module.activation_qtype is not None


def _own_output_scale(module: torch.nn.Module, input, output):
    """Forward hook that runs after a calibrated module's quantize_output hook.

    quantize_output wraps the module's `output_scale` buffer itself.  The in-place update would then rewrite the scale of
    every output already handed out at the module's next call (a module applied twice in one forward, an output kept
    across batches), where the reference rebinds the buffer and its earlier outputs keep their scale.  So the output
    gets a copy of the scale as it is now."""
    if isinstance(output, ActivationQBytesTensor) and output._scale is module.output_scale:
        return ActivationQBytesTensor(output.qtype, output.size(), output.stride(), output._data, output._scale.clone())
    return None


class Calibration(TorchFunctionMode):
    """Calibrate the activation scales of the quantized modules run inside it.

    Each forward of a quantized module with activations updates its scales with the absmax of the float activation:
    `scale = new` while the scale is exactly 1, `momentum * scale + new * (1 - momentum)` afterwards.

    Args:
        momentum (`float`): the momentum of the output-scale update.  The input scale always uses 0.9, as in the
            reference.
        streamline (`bool`): once a module that is not itself calibrated finishes its forward, remove the output
            quantization of each of its calibrated children (the reference's decisions; DESIGN.md, calibration quirks).
        debug (`bool`): print each quantized child's activation qtype and output scale after its parent has run.
    """

    def __init__(self, *args, momentum: float = 0.9, streamline=True, debug=False, **kwargs):
        super().__init__(*args, **kwargs)
        self.momentum, self.streamline, self.debug = momentum, streamline, debug
        self._global_hooks = []
        self._output_hooks = {}  # calibrated module -> handle of its _own_output_scale hook

    def __torch_function__(self, func, types, args=(), kwargs=None):
        # the mode marks the region being calibrated; every torch function inside it runs unchanged
        return func(*args, **(kwargs or {}))

    def __enter__(self):
        global _entered
        super().__enter__()
        _entered += 1
        # global hooks run before each module's own hooks: the input before quantize_input, the output before
        # quantize_output
        self._global_hooks = [register_module_forward_pre_hook(self.calibrate_input),
                              register_module_forward_hook(self.calibrate_output)]

    def __exit__(self, exc_type, exc_val, exc_tb):
        global _entered
        super().__exit__(exc_type, exc_val, exc_tb)
        _entered -= 1
        for handle in self._global_hooks + list(self._output_hooks.values()):
            handle.remove()
        self._global_hooks, self._output_hooks = [], {}

    def calibrate_input(self, module: torch.nn.Module, args):
        """Global forward pre-hook: update the input scale of a calibrated module.  Like the reference's hook it returns
        the first argument alone, which becomes the module's only argument."""
        if not _is_calibrated(module):
            return None
        x = args[0]
        if isinstance(x, ActivationQBytesTensor):
            _adopt_input_scale(module, torch.max(x._scale))
        else:
            _calibrate_scale(module, "input_scale", x, module.activation_qtype, _INPUT_MOMENTUM)
        if module not in self._output_hooks:
            self._output_hooks[module] = module.register_forward_hook(_own_output_scale)
        return x

    def calibrate_output(self, module: torch.nn.Module, input, output):
        """Global forward hook: update the output scale of a calibrated module from its float output; after any other
        module, apply streamline and debug to its children."""
        if _is_calibrated(module):
            _calibrate_scale(module, "output_scale", output, module.activation_qtype, self.momentum)
            return None
        if self.streamline:
            for child in module.children():
                if _is_calibrated(child):
                    child.disable_output_quantization()
        if self.debug:
            self._trace_children(module)
        return None

    @staticmethod
    def _trace_children(module: torch.nn.Module):
        from .nn import QModuleMixin

        for name, child in module.named_children():
            if not isinstance(child, QModuleMixin):
                continue
            if child.activation_qtype is None:
                state = "not quantized."
            else:
                state = f"quantized to {child.activation_qtype} with scale {child.output_scale}."
            print(f"{name}({type(child).__name__}) activations are {state}")
