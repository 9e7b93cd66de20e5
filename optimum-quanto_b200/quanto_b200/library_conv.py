"""The two `torch.ops.quanto.*` ops of the quantized 2-D convolution (the reference's QConv2d,
optimum/quanto/nn/qconv2d.py, whose forward is F.conv2d on a quantized weight):

  quanto::qbits_conv2d   F.conv2d with a packed int4 weight [Cout, Cin, kh, kw] quantized along axis 0
  quanto::qbytes_conv2d  F.conv2d with an int8 / float8 weight, weight-only (16-bit activations)

Both run as one implicit-GEMM launch on the tensor cores (csrc/conv_tc.cuh): the weight is read in its frozen storage,
which is byte for byte that of the linear weight [Cout, Cin * kh * kw], and dequantised in-kernel exactly as
`dequantize()` does; no im2col buffer and no dense weight is written.  Zero padding, stride and dilation, groups == 1,
NCHW-contiguous bf16 / fp16 input (batched [B, C, H, W] or unbatched [C, H, W]); the output is contiguous NCHW.
The result is rnd(conv + bias), the bias added to the fp32 sum and rounded once with it: what the reference's QConv2d
computes on the CPU, bit for bit (ATen's CUDA path rounds twice: cuDNN's output, then the bias add).

Defined here rather than in library.py so that each module registers and fakes exactly the ops it defines.  As there,
only the CUDA dispatch key gets a kernel and every op has a fake implementation for torch.compile.  `qbits_conv2d_ok`
and `qbytes_conv2d_ok` say which problems the weight tensors send to the kernel: those it takes whose reduction is
short enough for the kernel to beat the dequantize + F.conv2d composition (NATIVE_MAX_K); everything else runs that
composition.
"""
from typing import List

import torch

from . import _native as N
from .library import _bind_cuda, _define, _lib

__all__ = ["qbits_conv2d_ok", "qbytes_conv2d_ok", "native_conv2d"]

_define("qbits_conv2d", "(Tensor input, Tensor packed, Tensor scale, Tensor shift, Tensor? bias, int[] weight_shape, "
                        "int group_size, int bits, int[] stride, int[] padding, int[] dilation) -> Tensor")
_define("qbytes_conv2d", "(Tensor input, Tensor weights, Tensor scales, Tensor? bias, int[] stride, int[] padding, "
                         "int[] dilation) -> Tensor")

_HALF = (torch.float16, torch.bfloat16)
_BYTES = (torch.int8, torch.float8_e4m3fn, torch.float8_e5m2, torch.float8_e4m3fnuz)


def _pair(v, what: str) -> List[int]:
    v = list(v)
    if len(v) == 1:
        v = v * 2
    if len(v) != 2:
        raise ValueError(f"conv2d: {what} must have one or two values (got {v})")
    return [int(e) for e in v]


def _conv_geometry(input, weight_shape, stride, padding, dilation):
    """Shared checks of both ops -> (output shape, (stride, padding, dilation) as pairs)."""
    if len(weight_shape) != 4:
        raise ValueError(f"conv2d expects a weight [Cout, Cin, kh, kw] (got {list(weight_shape)})")
    if input.ndim not in (3, 4):
        raise ValueError(f"conv2d expects an input [B, C, H, W] or [C, H, W] (got {tuple(input.shape)})")
    if input.dtype not in _HALF:
        raise ValueError(f"conv2d: no sm_90a kernel for activations of dtype {input.dtype}")
    cout, cin, kh, kw = (int(e) for e in weight_shape)
    c, h, w = input.shape[-3:]
    if c != cin:
        raise ValueError(f"conv2d: input has {c} channels, the weight expects {cin} (groups == 1)")
    s, p, d = _pair(stride, "stride"), _pair(padding, "padding"), _pair(dilation, "dilation")
    if min(s) < 1 or min(d) < 1 or min(p) < 0:
        raise ValueError("conv2d: stride and dilation must be >= 1, padding >= 0")
    ho = (h + 2 * p[0] - d[0] * (kh - 1) - 1) // s[0] + 1
    wo = (w + 2 * p[1] - d[1] * (kw - 1) - 1) // s[1] + 1
    if ho <= 0 or wo <= 0:
        raise ValueError("conv2d: the kernel is larger than the padded input")
    shape = (cout, ho, wo) if input.ndim == 3 else (input.shape[0], cout, ho, wo)
    return shape, (s, p, d)


def _check_bias(bias, input, cout: int, what: str):
    if bias is not None and (bias.dtype != input.dtype or bias.numel() != cout):
        raise ValueError(f"{what}: bias must hold {cout} values of the input dtype")


# -------------------------------------------------------------------------------------------- qbits_conv2d
def _check_qbits_conv2d(input, packed, scale, shift, bias, weight_shape, group_size, bits, stride, padding, dilation):
    shape, geo = _conv_geometry(input, weight_shape, stride, padding, dilation)
    cout = int(weight_shape[0])
    k = int(weight_shape[1]) * int(weight_shape[2]) * int(weight_shape[3])
    if packed.dtype != torch.uint8:
        raise ValueError("qbits_conv2d: packed weights must be uint8")
    if scale.dtype != input.dtype:
        raise ValueError(f"qbits_conv2d: scale dtype {scale.dtype} does not match the activations ({input.dtype})")
    if shift.dtype.is_floating_point:
        if shift.dtype != input.dtype:
            raise ValueError(f"qbits_conv2d: float shift of dtype {shift.dtype} does not match the activations")
    elif shift.dtype not in (torch.uint8, torch.int8):
        raise ValueError("qbits_conv2d: integer shifts must be uint8 / int8 zero-points")
    if bits != 4:
        raise ValueError("qbits_conv2d: bits must be 4")
    if group_size <= 0 or k % group_size != 0:
        raise ValueError(f"qbits_conv2d: group size {group_size} does not divide Cin * kh * kw = {k}")
    rows = cout * (k // group_size)
    if scale.numel() != rows or shift.numel() != rows:
        raise ValueError("qbits_conv2d: scale / shift must hold one value per (out-channel, group)")
    if packed.numel() != -(-rows // 2) * group_size:
        raise ValueError("qbits_conv2d: packed tensor does not match the weight shape")
    _check_bias(bias, input, cout, "qbits_conv2d")
    return shape, geo


def qbits_conv2d_cuda(input, packed, scale, shift, bias, weight_shape: List[int], group_size: int, bits: int,
                      stride: List[int], padding: List[int], dilation: List[int]) -> torch.Tensor:
    shape, (s, p, d) = _check_qbits_conv2d(input, packed, scale, shift, bias, weight_shape, group_size, bits, stride,
                                           padding, dilation)
    x = input.reshape((1,) + tuple(input.shape)) if input.ndim == 3 else input
    x = x.contiguous()
    cout, cin, kh, kw = (int(e) for e in weight_shape)
    packed = packed.contiguous()
    scale_f = scale.reshape(-1).contiguous()
    shift_f = shift.reshape(-1).contiguous()
    shift_is_int = 0 if shift_f.dtype.is_floating_point else 1
    if shift_f.dtype == torch.int8:
        shift_f = shift_f.view(torch.uint8)
    bias_f = None if bias is None else bias.reshape(-1).contiguous()
    out = torch.empty(shape, dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device):
        lib = N.load()
        N.check(lib.qb200_qbits_conv2d(N.ptr(x), N.ptr(packed), N.ptr(scale_f), N.ptr(shift_f), N.ptr(bias_f),
                                       N.ptr(out), x.shape[0], cin, x.shape[2], x.shape[3], cout, kh, kw, s[0], s[1],
                                       p[0], p[1], d[0], d[1], group_size, bits, N.DTYPE_CODE[x.dtype], shift_is_int,
                                       N.stream_ptr(x.device)), "quanto::qbits_conv2d")
    return out


# ------------------------------------------------------------------------------------------- qbytes_conv2d
def _check_qbytes_conv2d(input, weights, scales, bias, stride, padding, dilation):
    shape, geo = _conv_geometry(input, weights.shape, stride, padding, dilation)
    if weights.dtype not in _BYTES:
        raise ValueError(f"qbytes_conv2d: no sm_90a kernel for weights of dtype {weights.dtype}")
    if scales.dtype != input.dtype or scales.numel() != weights.shape[0]:
        raise ValueError("qbytes_conv2d: scales must hold one value per out-channel, of the input dtype")
    _check_bias(bias, input, weights.shape[0], "qbytes_conv2d")
    return shape, geo


def qbytes_conv2d_cuda(input, weights, scales, bias, stride: List[int], padding: List[int],
                       dilation: List[int]) -> torch.Tensor:
    shape, (s, p, d) = _check_qbytes_conv2d(input, weights, scales, bias, stride, padding, dilation)
    x = input.reshape((1,) + tuple(input.shape)) if input.ndim == 3 else input
    x = x.contiguous()
    cout, cin, kh, kw = weights.shape
    w = weights.contiguous()
    scales_f = scales.reshape(-1).contiguous()
    bias_f = None if bias is None else bias.reshape(-1).contiguous()
    out = torch.empty(shape, dtype=x.dtype, device=x.device)
    with torch.cuda.device(x.device):
        lib = N.load()
        N.check(lib.qb200_qbytes_conv2d(N.ptr(x), N.ptr(w), N.ptr(scales_f), N.ptr(bias_f), N.ptr(out), x.shape[0],
                                        cin, x.shape[2], x.shape[3], cout, kh, kw, s[0], s[1], p[0], p[1], d[0], d[1],
                                        N.DTYPE_CODE[w.dtype], N.DTYPE_CODE[x.dtype], N.stream_ptr(x.device)),
                "quanto::qbytes_conv2d")
    return out


_bind_cuda("qbits_conv2d", qbits_conv2d_cuda)
_bind_cuda("qbytes_conv2d", qbytes_conv2d_cuda)


# ------------------------------------------------------------------------------- what the kernel takes
def _aligned16(t) -> bool:
    """The kernels read weight rows with 16-byte loads (the C ABI declines an unaligned weight).  A contiguous tensor is
    read in place, so its storage offset must keep the 16-byte alignment of its storage (the caching allocator's blocks
    are 512-byte aligned); any other tensor is copied to a fresh contiguous one by the op.  Checked on the offset, not on
    data_ptr(), so that the same predicate holds for the fake tensors of a traced graph."""
    return not t.is_contiguous() or (t.storage_offset() * t.element_size()) % 16 == 0


def _common_ok(input, cout: int, k: int, bias, stride, padding, dilation, groups) -> bool:
    """Problems both conv kernels take (beyond the weight): a plain CUDA bf16 / fp16 NCHW-contiguous input, groups == 1,
    integer padding, K % 16 == 0 and a bias of the input dtype."""
    from .tensor.qtensor import QTensor

    if isinstance(input, QTensor):
        return False  # a quantized (ActivationQBytesTensor) input: composition
    if isinstance(padding, str) or groups != 1:
        return False
    if not input.is_cuda or input.dtype not in _HALF or input.ndim not in (3, 4) or not input.is_contiguous():
        return False
    if bias is not None and (bias.dtype != input.dtype or bias.numel() != cout):
        return False
    return k % 16 == 0


def qbits_conv2d_ok(input, weight, bias, stride, padding, dilation, groups) -> bool:
    """Whether quanto::qbits_conv2d runs F.conv2d(input, weight, bias, ...) for a WeightQBitsTensor `weight`: axis-0
    packed int4 of the input dtype, Cout even, a group that is a multiple of 32 or per-axis."""
    if weight.ndim != 4 or weight._axis != 0 or weight._qtype.bits != 4 or not hasattr(weight._data, "_data"):
        return False
    cout, cin, kh, kw = weight.shape
    k = cin * kh * kw
    g = weight._group_size if weight._group_size is not None else k
    shift = weight._shift
    return (
        _common_ok(input, cout, k, bias, stride, padding, dilation, groups)
        and input.shape[-3] == cin
        and weight._data._data.is_cuda and _aligned16(weight._data._data)
        and weight._scale.dtype == input.dtype
        and (shift.dtype in (torch.uint8, torch.int8) or shift.dtype == input.dtype)
        and cout % 2 == 0 and (g % 32 == 0 or g == k) and k % g == 0
        and weight._scale.numel() == cout * (k // g)
        and _conv_out_ok(input, weight.shape, stride, padding, dilation)
    )


def qbytes_conv2d_ok(input, weight, bias, stride, padding, dilation, groups) -> bool:
    """Whether quanto::qbytes_conv2d runs F.conv2d(input, weight, bias, ...) for a WeightQBytesTensor `weight`: axis-0
    int8 / float8 weights with one scale per out-channel of the input dtype."""
    if weight.ndim != 4 or weight._axis != 0 or weight._data.dtype not in _BYTES:
        return False
    cout, cin, kh, kw = weight.shape
    return (
        _common_ok(input, cout, cin * kh * kw, bias, stride, padding, dilation, groups)
        and input.shape[-3] == cin
        and weight._data.is_cuda and _aligned16(weight._data)
        and weight._scale.dtype == input.dtype and weight._scale.numel() == cout
        and _conv_out_ok(input, weight.shape, stride, padding, dilation)
    )


# Routing rule on the shape, from GPU time (DESIGN 6: CUDA-graph replays, H100).  The kernel costs about 4 us of GPU
# time per 64-k pipeline stage of a tile wave, and knocking out its gather loads or its output stores does not change
# that, while dequantize() + cuDNN costs tens of microseconds in all.  The kernel only wins when the reduction is a
# single stage: K = Cin * kh * kw <= 64 (1.2x on a 1x1 conv with Cin 64); every measured conv with a larger K is 1.7-9x
# slower on the kernel, so it takes the composition.  The rule targets GPU time, what a captured or compiled model pays
# and what bounds any model whose host runs ahead; an eager model of small convs pays more in host dispatch for the
# composition's launches (the eager columns of tools/bench_qconv2d.py), which capturing it removes.
NATIVE_MAX_K = 64


def _conv_out_ok(input, weight_shape, stride, padding, dilation) -> bool:
    """The geometry is valid, fits the C ABI, and the reduction is short enough for the kernel to beat the composition."""
    try:
        shape, _ = _conv_geometry(input, weight_shape, stride, padding, dilation)
    except ValueError:
        return False
    cout, cin, kh, kw = (int(e) for e in weight_shape)
    pixels = shape[-1] * shape[-2] * (shape[0] if len(shape) == 4 else 1)
    if pixels > _INT32_MAX or cin * kh * kw > _INT32_MAX or max(input.shape[-2:]) > _INT32_MAX // 2:
        return False  # the C ABI declines dimensions over int32
    return cin * kh * kw <= NATIVE_MAX_K


_INT32_MAX = 2 ** 31 - 1


def conv2d_args(input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
    """The arguments of F.conv2d, by name."""
    return input, weight, bias, stride, padding, dilation, groups


def _as_pair(v):
    return [int(v), int(v)] if isinstance(v, int) else [int(e) for e in v]


def native_conv2d(args, kwargs, qbits_cls, qbytes_cls):
    """F.conv2d(*args, **kwargs) on a quantized weight as one quanto::qbits_conv2d / quanto::qbytes_conv2d launch, or
    None: the caller then runs the composition (`dequantize()` + aten.convolution through qfallback), the reference's
    behaviour.  The kernel runs when no graph is needed (a frozen weight, or no_grad) and the predicates above take the
    problem: fp32, grouped / depthwise convs, quantized or channels_last inputs, string paddings, what the C ABI
    declines and convolutions beyond the routing rule take the composition.  `qbits_cls` / `qbytes_cls`: the weight
    classes, this package's or the reference's (integration.bind_reference)."""
    input, weight, bias, stride, padding, dilation, groups = conv2d_args(*args, **kwargs)
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (input, weight, bias)):
        return None
    if isinstance(padding, str):
        return None
    stride, padding, dilation = _as_pair(stride), _as_pair(padding), _as_pair(dilation)
    if type(weight) is qbits_cls and qbits_conv2d_ok(input, weight, bias, stride, padding, dilation, groups):
        cout, cin, kh, kw = weight.shape
        group = weight._group_size if weight._group_size is not None else cin * kh * kw
        return torch.ops.quanto.qbits_conv2d(input, weight._data._data, weight._scale, weight._shift, bias,
                                             list(weight.shape), group, weight._qtype.bits, stride, padding, dilation)
    if type(weight) is qbytes_cls and qbytes_conv2d_ok(input, weight, bias, stride, padding, dilation, groups):
        return torch.ops.quanto.qbytes_conv2d(input, weight._data, weight._scale, bias, stride, padding, dilation)
    return None


# ------------------------------------------------------------------------------------------ fake implementations
def _qbits_conv2d_fake(input, packed, scale, shift, bias, weight_shape, group_size, bits, stride, padding, dilation):
    shape, _ = _check_qbits_conv2d(input, packed, scale, shift, bias, weight_shape, group_size, bits, stride, padding,
                                   dilation)
    return input.new_empty(shape)


def _qbytes_conv2d_fake(input, weights, scales, bias, stride, padding, dilation):
    shape, _ = _check_qbytes_conv2d(input, weights, scales, bias, stride, padding, dilation)
    return input.new_empty(shape)


FAKE_IMPLS = {
    "qbits_conv2d": _qbits_conv2d_fake,
    "qbytes_conv2d": _qbytes_conv2d_fake,
}
for _name, _fake in FAKE_IMPLS.items():
    torch.library.register_fake("quanto::" + _name, _fake, lib=_lib)
