"""Autograd functions of the quantized linear (forward and input gradient on the native kernels).

Mirrors optimum/quanto/tensor/function.py:21-63 (QuantizedLinearFunction) and
optimum/quanto/tensor/weights/qbytes.py:68-82 (WeightQBytesLinearFunction).  The input gradient gO @ W of the int4 and
8-bit linears reads the quantized weights (`quanto::qbits_grad_input` / `quanto::qbytes_grad_input`) instead of
dequantising a dense copy of the weight for a dense GEMM; the weight and bias gradients keep the base formulas.
"""
import torch

from .qtensor import QBytesTensor

__all__ = ["QuantizedLinearFunction", "WeightQBytesLinearFunction", "WeightQBitsLinearFunction", "linear_backward",
           "qbits_grad_input", "qbytes_grad_input", "NATIVE_GRAD_INPUT_MAX_M"]

# Route selection of the input gradient: the native kernel up to this many gradient rows, the composition (dequantize +
# dense GEMM) above.  Measured with tools/bench_grad_input.py on an H100 80GB HBM3 at 700 W (DESIGN.md section 6): at
# M <= 128 the kernel is up to 2.4x faster than the composition (0.8-0.95x where K = 4096 leaves only 32 column tiles);
# from M = 512 on cuBLAS on the dequantised copy is mostly faster, by up to 2x at M = 4096.
NATIVE_GRAD_INPUT_MAX_M = 128


def linear_backward(ctx, gO, grad_input):
    """QuantizedLinearFunction.backward with the input gradient taken from `grad_input(gO_2d, other)` ([M, N] -> [M, K],
    or None for the base formula `torch.matmul(gO, other)`).  The weight and bias gradients are the base formulas."""
    input, other = ctx.saved_tensors
    out_features, in_features = other.shape
    g_in = g_w = g_b = None
    if ctx.needs_input_grad[0]:
        g2 = grad_input(gO.reshape(-1, out_features), other) if gO.numel() > 0 else None
        g_in = torch.matmul(gO, other) if g2 is None else g2.reshape(gO.shape[:-1] + (in_features,))
    if ctx.needs_input_grad[1]:
        g_w = torch.matmul(gO.reshape(-1, out_features).t(), input.reshape(-1, in_features))
    if ctx.needs_input_grad[2]:
        g_b = gO.sum(tuple(range(gO.ndim - 1)))
    return g_in, g_w, g_b


def qbits_grad_input(gO, other):
    """gO [M, N] @ dequant(other) for an axis-0 packed weight on CUDA whose dtype is the gradient's; else None."""
    if gO.shape[0] > NATIVE_GRAD_INPUT_MAX_M:
        return None
    data = getattr(other, "_data", None)
    packed = getattr(data, "_data", None)
    if packed is None or not hasattr(data, "_bits") or not packed.is_cuda or len(other.shape) != 2:
        return None
    n, k = other.shape
    g = other._group_size
    if (other._axis != 0 or g is None or g % 4 != 0 or k % g != 0 or other._scale.numel() != n * (k // g)
            or gO.dtype != other._scale.dtype or gO.device != packed.device
            or not (other._shift.dtype in (torch.uint8, torch.int8) or other._shift.dtype == other._scale.dtype)):
        return None
    return torch.ops.quanto.qbits_grad_input(gO, packed, other._scale, other._shift, n, g, data._bits)


def qbytes_grad_input(gO, other):
    """gO [M, N] @ (scale * data) for an 8-bit weight [N, K] on CUDA whose scale dtype is the gradient's; else None."""
    if gO.shape[0] > NATIVE_GRAD_INPUT_MAX_M:
        return None
    data, scale = other._data, other._scale
    if (not data.is_cuda or data.ndim != 2 or other._axis not in (0, None) or gO.dtype != scale.dtype
            or gO.device != data.device or scale.numel() not in (1, data.shape[0])):
        return None
    return torch.ops.quanto.qbytes_grad_input(gO, data, scale)


class QuantizedLinearFunction(torch.autograd.Function):
    """Generic quantized linear: dequantise `other` and multiply (the reference's base path)."""

    @staticmethod
    def forward(ctx, input, other, bias=None):
        ctx.save_for_backward(input, other)
        output = torch.matmul(input, other.t())
        if bias is not None:
            output = output + bias
        return output

    @staticmethod
    def backward(ctx, gO):
        input, other = ctx.saved_tensors
        out_features, in_features = other.shape
        g_in = g_w = g_b = None
        if ctx.needs_input_grad[0]:
            g_in = torch.matmul(gO, other)
        if ctx.needs_input_grad[1]:
            g_w = torch.matmul(gO.reshape(-1, out_features).t(), input.reshape(-1, in_features))
        if ctx.needs_input_grad[2]:
            g_b = gO.sum(tuple(range(gO.ndim - 1)))
        return g_in, g_w, g_b


class WeightQBytesLinearFunction(QuantizedLinearFunction):
    """8-bit weights: one `quanto::qbytes_mm` call; with quantized activations the scales are multiplied first."""

    @staticmethod
    def forward(ctx, input, other, bias=None):
        ctx.save_for_backward(input, other)
        # with a bias: quanto::qbytes_linear = the same kernel with the bias added in its epilogue (one launch less and
        # no extra pass over [M, N]); same rounding order as `qbytes_mm(...) + bias`
        if isinstance(input, QBytesTensor):
            scales = input._scale * other._scale
            if bias is not None:
                return torch.ops.quanto.qbytes_linear(input._data, other._data, scales, bias)
            return torch.ops.quanto.qbytes_mm(input._data, other._data, scales)
        k = input.shape[-1]
        if bias is not None:
            output = torch.ops.quanto.qbytes_linear(input.reshape(-1, k), other._data, other._scale, bias)
        else:
            output = torch.ops.quanto.qbytes_mm(input.reshape(-1, k), other._data, other._scale)
        return output.reshape(input.shape[:-1] + (other.shape[0],))

    @staticmethod
    def backward(ctx, gO):
        return linear_backward(ctx, gO, qbytes_grad_input)


class WeightQBitsLinearFunction(QuantizedLinearFunction):
    """Packed int4 / int2 weights in canonical axis-0 storage: one fused `quanto::qbits_mm` launch (bias included)."""

    @staticmethod
    def forward(ctx, input, other, bias=None):
        ctx.save_for_backward(input, other)
        if isinstance(input, QBytesTensor):
            input = input.dequantize()  # the int4 GEMM always sees float activations (SURVEY 3.1)
        n, k = other.shape
        group = other._group_size if other._group_size is not None else k  # per-axis = one group per out-feature
        out = torch.ops.quanto.qbits_mm(
            input.reshape(-1, k), other._data._data, other._scale, other._shift, bias, n, group, other._qtype.bits
        )
        return out.reshape(input.shape[:-1] + (n,))

    @staticmethod
    def backward(ctx, gO):
        return linear_backward(ctx, gO, qbits_grad_input)
