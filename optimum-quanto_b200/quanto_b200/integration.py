"""Bind the sm_90a kernels into the REAL `optimum.quanto` package (the binding INTEGRATION.md describes, executable).

    import optimum.quanto                      # the reference, unmodified
    from quanto_b200.integration import bind_reference
    bind_reference()

After this, every `optimum.quanto` object keeps working as before -- `quantize()`, `freeze()`, `QLinear`,
`WeightQBitsTensor`, state dicts -- and the quantized-linear forward on a CUDA (sm_90) device runs on this library:

1. op registry: `quanto::unpack`, `quanto::quantize_symmetric`, `quanto::qbytes_mm` (and `quanto::quantize_affine`) get
   this library's CUDA implementations (importing `quanto_b200.library` after the reference re-binds the CUDA dispatch key;
   optimum/quanto/library/extensions/cuda/__init__.py:77-79, library/qbytes_mm.py:73).  The retired external-kernel ops
   (`gemm_f16i4_awq`, `gemm_f16i4_marlin`, `gemm_f16f8_marlin`, `pack_fp8_marlin`, cuda/__init__.py:82-202) are simply no
   longer reached;
2. `WeightQBitsTensor.create` / `WeightQBytesTensor.create` (tensor/weights/qbits.py:67-138, qbytes.py:87-143) stop routing
   CUDA tensors to the AWQ / TinyGemm / Marlin-FP8 repacking subclasses: the kernels read the canonical packing, so
   `create()` returns the canonical tensor and nothing is repacked at `freeze()` / `.to(device)` / load time;
3. `F.linear(x, WeightQBitsTensor)` on CUDA calls `quanto::qbits_mm` -- ONE fused launch instead of
   unpack + scale + shift + ungroup + matmul (tensor/weights/qbits.py:262-281, tensor/function.py:42-47); its backward
   takes the input gradient from `quanto::qbits_grad_input` (one launch that reads the packed weights, instead of
   `torch.matmul(gO, other)` on a dequantised dense copy) and keeps the reference's weight and bias gradients;
4. `WeightQBytesLinearFunction.forward` (tensor/weights/qbytes.py:68-82) keeps calling `quanto::qbytes_mm`, with the bias
   fused into the kernel epilogue when there is one; its backward takes the input gradient from
   `quanto::qbytes_grad_input` the same way;
5. `HqqOptimizer.__call__` (tensor/optimizers/hqq_optimizer.py:60-87 after affine_optimizer.py:27-64) runs
   `quanto::quantize_qbits_hqq` -- two launches, no host synchronisation -- for a CUDA bf16 / fp16 weight quantized along
   axis 0 to qint4 / qint2, and the reference's own code for everything else and whatever the kernel declines;
6. `aten.bmm` and `aten._softmax` of the reference's `ActivationQBytesTensor` table
   (tensor/activations/qbytes_ops.py:175-186, 208-215) run on `quanto::qbytes_bmm` (an exact int8 x int8 product on the
   tensor cores instead of an fp32 bmm of int8 values cast to fp32) and `quanto::qbytes_softmax` (codes in, codes out,
   one launch) for CUDA tensors; every case those entries decline falls through to the reference's own entry;
7. `F.conv2d` on the reference's `WeightQBitsTensor` / `WeightQBytesTensor` (its QConv2d, optimum/quanto/nn/qconv2d.py)
   runs `quanto::qbits_conv2d` / `quanto::qbytes_conv2d` -- one implicit-GEMM launch -- when no graph is needed and the
   kernel takes the problem, instead of qfallback's dense dequantised copy + cuDNN; everything else keeps the
   reference's route.
8. the reference's `QLayerNorm` (optimum/quanto/nn/qlayernorm.py) runs `quanto::qbytes_layer_norm` -- the layer norm
   and its output quantisation in one launch, from floats or codes -- under the conditions of the package's QLayerNorm
   (library_norm.qlayernorm_forward), except while a `Calibration` mode is active; its quantize_output hook passes the
   op's codes through instead of quantizing them again.

Used by tools/run_reference_tests.py to run the reference's OWN hot-path tests (tests/library, tests/tensor/ops,
tests/nn/test_qlinear.py, and for 6 tests/tensor/ops/test_mm_dispatch.py, tests/tensor/activations/test_activations_dispatch.py,
tests/nn/test_qattention.py, for 7 tests/nn/test_qconv2d.py, for 8 tests/nn/test_qlayernorm.py) against these kernels.  Nothing here is imported by the rest of the package.
"""
import torch

__all__ = ["bind_reference"]

_bound = False


def bind_reference():
    global _bound
    if _bound:
        return
    import optimum.quanto  # noqa: F401  (must be imported first: it DEFINES the quanto:: ops)
    from optimum.quanto.tensor import function as ref_function
    from optimum.quanto.tensor.qbytes import QBytesTensor as RefQBytesTensor
    from optimum.quanto.tensor.weights import qbits as ref_qbits
    from optimum.quanto.tensor.weights import qbytes as ref_qbytes

    from . import library  # noqa: F401  (re-binds the CUDA dispatch key of the shared ops, defines the fused ones)
    from .tensor.function import linear_backward, qbits_grad_input, qbytes_grad_input

    RefQBits = ref_qbits.WeightQBitsTensor
    RefQBytesW = ref_qbytes.WeightQBytesTensor

    # ---- 2. create(): canonical tensors on CUDA (CPU / other devices keep the reference's routing)
    orig_qbits_create = RefQBits.create
    orig_qbytes_create = RefQBytesW.create

    def qbits_create(qtype, axis, group_size, size, stride, data, scale, shift, requires_grad=False):
        if data.device.type == "cuda":
            return RefQBits(qtype, axis, group_size, size, stride, data, scale, shift, requires_grad)
        return orig_qbits_create(qtype, axis, group_size, size, stride, data, scale, shift, requires_grad)

    def qbytes_create(qtype, axis, size, stride, data, scale, activation_qtype=None, requires_grad=False):
        if data.device.type == "cuda":
            return RefQBytesW(qtype, axis, size, stride, data, scale, activation_qtype, requires_grad)
        return orig_qbytes_create(qtype, axis, size, stride, data, scale, activation_qtype, requires_grad)

    RefQBits.create = staticmethod(qbits_create)
    RefQBytesW.create = staticmethod(qbytes_create)

    # ---- 3. fused int4 / int2 linear
    class FusedQBitsLinear(ref_function.QuantizedLinearFunction):
        @staticmethod
        def forward(ctx, input, other, bias=None):
            ctx.save_for_backward(input, other)
            if isinstance(input, RefQBytesTensor):
                input = input.dequantize()
            n, k = other.shape
            group = other._group_size if other._group_size is not None else k
            out = torch.ops.quanto.qbits_mm(input.reshape(-1, k), other._data._data, other._scale, other._shift, bias, n,
                                            group, other._qtype.bits)
            return out.reshape(input.shape[:-1] + (n,))

        @staticmethod
        def backward(ctx, gO):
            return linear_backward(ctx, gO, qbits_grad_input)

    def fused_ok(w, x):
        from optimum.quanto.tensor.packed import PackedTensor
        if type(w) is not RefQBits or len(w.shape) != 2 or not isinstance(w._data, PackedTensor):
            return False
        n, k = w.shape
        g = w._group_size if w._group_size is not None else k
        in_dtype = x._scale.dtype if isinstance(x, RefQBytesTensor) else x.dtype
        return (w._axis == 0 and w._data._data.is_cuda and w._qtype.bits in (2, 4)
                and w._scale.dtype in (torch.float32, torch.float16, torch.bfloat16)
                and (w._shift.dtype in (torch.uint8, torch.int8) or w._shift.dtype == w._scale.dtype)
                and k % g == 0 and w._scale.numel() == n * (k // g) and in_dtype == w._scale.dtype)

    orig_tf = RefQBits.__torch_function__.__func__

    def qbits_torch_function(cls, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func is torch.nn.functional.linear:
            def split(input, other, bias=None):
                return input, other, bias
            input, other, bias = split(*args, **kwargs)
            if fused_ok(other, input):
                return FusedQBitsLinear.apply(input, other, bias)
        return orig_tf(cls, func, types, args, kwargs)

    RefQBits.__torch_function__ = classmethod(qbits_torch_function)

    # ---- 4. 8-bit linear: bias fused into the qbytes_mm epilogue
    class FusedQBytesLinear(ref_function.QuantizedLinearFunction):
        @staticmethod
        def forward(ctx, input, other, bias=None):
            ctx.save_for_backward(input, other)
            if isinstance(input, RefQBytesTensor):
                scales = input._scale * other._scale
                data = input._data
            else:
                scales, data = other._scale, input.reshape(-1, input.shape[-1])
            if bias is not None and data.is_cuda:
                out = torch.ops.quanto.qbytes_linear(data, other._data, scales, bias)
            else:
                out = torch.ops.quanto.qbytes_mm(data, other._data, scales)
                if bias is not None:
                    out = out + bias
            return out.reshape(input.shape[:-1] + (other.shape[0],))

        @staticmethod
        def backward(ctx, gO):
            return linear_backward(ctx, gO, qbytes_grad_input)

    ref_qbytes.WeightQBytesLinearFunction = FusedQBytesLinear

    # ---- 5. HQQ shift search on the device
    from optimum.quanto.tensor.optimizers import HqqOptimizer as RefHqq

    from .tensor.optimizers import HqqOptimizer
    from .tensor.qtype import qint2, qint4

    orig_hqq_call = RefHqq.__call__

    def hqq_call(self, base, qtype, axis, group_size=None, zeropoint=False):
        qt = {2: qint2, 4: qint4}.get(qtype.bits) if qtype.name in ("qint2", "qint4") else None
        if qt is not None:
            opt = HqqOptimizer(self.lp_norm, self.beta, self.kappa, self.iters, self.verbose)
            fused = opt.fused(base, qt, axis, group_size, zeropoint)
            if fused is not None:
                return fused[1], fused[2]
        return orig_hqq_call(self, base, qtype, axis, group_size, zeropoint)

    RefHqq.__call__ = hqq_call

    # ---- 6. quantized attention: int8 bmm and softmax of per-tensor activations
    from optimum.quanto.tensor.activations import qbytes_ops as ref_ops
    from optimum.quanto.tensor.activations.qbytes import ActivationQBytesTensor as RefActivation
    from optimum.quanto.tensor.core import dtype_info as ref_dtype_info
    from optimum.quanto.tensor.qtype import qint8 as ref_qint8

    from . import library_attention  # noqa: F401  (defines quanto::qbytes_bmm / quanto::qbytes_softmax)

    aten = torch.ops.aten
    table = ref_ops._QBYTESTENSOR_OP_TABLE
    orig_bmm, orig_softmax = table[aten.bmm], table[aten._softmax]

    def per_tensor(t):
        return isinstance(t, RefActivation) and t.axis is None and t._data.is_cuda and t._scale.numel() == 1

    def bmm(input, other):
        if (per_tensor(input) and per_tensor(other) and input.qtype == ref_qint8 and other.qtype == ref_qint8
                and other._scale.dtype == input._scale.dtype):
            return torch.ops.quanto.qbytes_bmm(input._data, other._data, input._scale, other._scale)
        return orig_bmm(input, other)

    def softmax(input, dim, half_to_float):
        if per_tensor(input) and not half_to_float and dim in (-1, input.ndim - 1):
            out_scale = torch.tensor(1 / ref_dtype_info(input.qtype.dtype).max, dtype=input._scale.dtype).to(
                input.device)
            data = torch.ops.quanto.qbytes_softmax(input._data, input._scale, out_scale)
            return RefActivation(input.qtype, data.size(), data.stride(), data, out_scale)
        return orig_softmax(input, dim, half_to_float)

    table[aten.bmm] = bmm
    table[aten._softmax] = softmax

    # ---- 7. quantized conv2d: the package's own routing (library_conv.native_conv2d), for the reference's classes
    from . import library_conv

    def conv_torch_function(orig):
        def torch_function(cls, func, types, args=(), kwargs=None):
            if func is torch.nn.functional.conv2d:
                out = library_conv.native_conv2d(args, kwargs or {}, RefQBits, RefQBytesW)
                if out is not None:
                    return out
            return orig(cls, func, types, args, kwargs)
        return classmethod(torch_function)

    RefQBits.__torch_function__ = conv_torch_function(RefQBits.__torch_function__.__func__)
    RefQBytesW.__torch_function__ = conv_torch_function(RefQBytesW.__torch_function__.__func__)

    # ---- 8. QLayerNorm: the layer norm and its output quantisation in one launch (library_norm.qlayernorm_forward)
    from optimum.quanto.calibrate import Calibration as RefCalibration
    from optimum.quanto.nn import qmodule as ref_qmodule
    from optimum.quanto.nn.qlayernorm import QLayerNorm as RefQLayerNorm

    from . import library_norm

    orig_ln_forward = RefQLayerNorm.forward

    def ln_forward(self, input):
        # calibrate_output must see the float output: keep the composition while a Calibration mode is active
        if not any(isinstance(m, RefCalibration) for m in torch.overrides._get_current_function_mode_stack()):
            # the reference's disable_output_quantization removes the hook but keeps its handle
            handle = self._quantize_hooks.get("output")
            live = handle is not None and handle.id in self._forward_hooks
            out = library_norm.qlayernorm_forward(self, input, RefActivation, live)
            if out is not None:
                return out
        return orig_ln_forward(self, input)

    RefQLayerNorm.forward = ln_forward
    orig_quantize_activation = ref_qmodule.quantize_activation

    def quantize_activation(t, qtype, scale):
        # the quantize_output hook of a QLayerNorm that returned the op's codes with this very scale: nothing to do
        if isinstance(t, RefActivation) and t.qtype == qtype and t._scale is scale:
            return t
        return orig_quantize_activation(t, qtype=qtype, scale=scale)

    ref_qmodule.quantize_activation = quantize_activation
    _bound = True
