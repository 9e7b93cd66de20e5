"""Quantized 2-D convolution on the GPU: quanto::qbits_conv2d / quanto::qbytes_conv2d under the parity contract of the
int4 / mixed GEMMs (DESIGN 4) on the im2col view, every instantiation, the routes that keep the dequantize + F.conv2d
composition, QConv2d end to end against the reference's fixture, the one-launch 4-D freeze and torch.compile."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from helpers import ROOT, band_rows, check_linear, make_qbits_weights, torch_to_bits
from oracle import conv_oracle as CO
from oracle import quanto_oracle as O

pytestmark = pytest.mark.gpu

if not torch.cuda.is_available():
    pytest.skip("needs a GPU", allow_module_level=True)

import quanto_b200 as q  # noqa: E402
from quanto_b200 import _native as N  # noqa: E402
from quanto_b200.tensor import ActivationQBytesTensor, WeightQBitsTensor, WeightQBytesTensor  # noqa: E402

DEV = torch.device("cuda:0")
DT = {"f16": torch.float16, "bf16": torch.bfloat16}
WDT = {"int8": torch.int8, "e4m3fn": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2, "e4m3fnuz": torch.float8_e4m3fnuz}
GOLDEN = os.path.join(ROOT, "tests", "golden", "qconv2d.npz")


def bits_t(arr, tag):
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.int16)).view(DT[tag]).to(DEV)


def make_input(b, c, h, w, tag, seed, border=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(b, c, h, w, generator=g)
    if border is not None:  # large border pixels: a gather that reads a padding tap from the image shows
        x[:, :, 0, :] = border
        x[:, :, -1, :] = border
        x[:, :, :, 0] = border
        x[:, :, :, -1] = border
    return x.to(DT[tag]).to(DEV)


def check_conv(y, x, wdeq, bias, tag, stride, padding, dilation, label):
    """y [B, Cout, Ho, Wo] against the float64 oracle of the im2col GEMM (sampled rows on large problems) and, in full,
    against fp32 F.conv2d of the same operands.  The kernel adds the bias to the fp32 sum and rounds once (the
    reference's QConv2d on the CPU): for the linear oracle the bias is one more k with activation 1."""
    cout, _, kh, kw = wdeq.shape
    xb = torch_to_bits(x)
    cols, (b, ho, wo) = CO.im2col(xb, kh, kw, stride, padding, dilation)
    wb = torch_to_bits(wdeq).reshape(cout, -1)
    if bias is not None:
        one = torch_to_bits(torch.ones(1, dtype=x.dtype))
        cols = np.concatenate([cols, np.broadcast_to(one, (cols.shape[0], 1))], axis=1)
        wb = np.concatenate([wb, torch_to_bits(bias).reshape(cout, 1)], axis=1)
    assert y.shape == (b, cout, ho, wo), (label, tuple(y.shape))
    assert y.is_contiguous()
    y_mk = y.permute(0, 2, 3, 1).reshape(-1, cout)
    m = y_mk.shape[0]
    rows = np.arange(m) if m * cout <= 1 << 16 else band_rows(m, seed=m)
    check_linear(y_mk[torch.from_numpy(rows).to(DEV)], cols[rows], wb, None, tag, label)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        ref = F.conv2d(x.float(), wdeq.float(), None if bias is None else bias.float(), stride, padding,
                       dilation).to(y.dtype)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    rel = float((y.float() - ref.float()).norm() / ref.float().norm())
    assert rel < 1e-3, (label, rel)


def qbits_weight(cout, k, group, tag, zp, seed):
    """(packed, scale, shift, dequantised [cout, k]) of a synthetic canonical int4 weight."""
    _, packed, scale, shift = make_qbits_weights(cout, k, group, tag, seed=seed, zeropoint=zp)
    deq = O.dequantize_qbits(packed, 4, scale, shift, tag, cout, k, group, shift_is_int=zp)
    packed_t = torch.from_numpy(packed).to(DEV)
    scale_t = bits_t(scale, tag).reshape(-1, 1)
    shift_t = torch.from_numpy(shift).to(DEV).reshape(-1, 1) if zp else bits_t(shift, tag).reshape(-1, 1)
    return packed_t, scale_t, shift_t, bits_t(deq, tag).reshape(cout, k)


def run_qbits(x, cout, kh, kw, group, tag, zp, bias, stride, padding, dilation, seed=0):
    cin = x.shape[-3]
    k = cin * kh * kw
    g = group or k
    packed, scale, shift, deq = qbits_weight(cout, k, g, tag, zp, seed)
    y = torch.ops.quanto.qbits_conv2d(x, packed, scale, shift, bias, [cout, cin, kh, kw], g, 4, list(stride),
                                      list(padding), list(dilation))
    return y, deq.reshape(cout, cin, kh, kw)


def make_bias(cout, tag, seed):
    g = torch.Generator().manual_seed(seed + 1000)
    return (torch.randn(cout, generator=g) * 0.5).to(DT[tag]).to(DEV)


# ------------------------------------------------------------------------------------------------ int4 grid
# (B, Cin, H, W, Cout, kh, stride, padding, dilation, group): M = B * Ho * Wo is never a multiple of the tile, so tiles
# straddle images and end ragged; Cout 96 / 200 leave the N tile partial
GEOMETRIES = [
    (2, 32, 9, 9, 96, 3, 1, 1, 1, 96),       # K = 288: group 96, K % 64 == 32 (the second set of the last stage)
    (1, 192, 7, 5, 64, 1, 1, 0, 1, 96),      # 1x1
    (5, 32, 6, 7, 96, 5, 1, 2, 1, 160),      # 5x5, padding 2, group 160 (two sets per stage)
    (2, 32, 11, 10, 200, 3, 2, 1, 1, 96),    # stride 2
    (2, 32, 12, 9, 64, 3, 1, 2, 2, 96),      # dilation 2
    (2, 48, 10, 11, 64, 3, 2, 0, 2, None),   # K = 432 per-axis: a K tail of 48
    (1, 128, 8, 8, 96, 3, 1, 1, 1, 32),
    (2, 128, 8, 8, 96, 3, 1, 1, 1, 64),
    (2, 128, 8, 8, 96, 3, 1, 1, 1, 128),
    (2, 128, 8, 8, 96, 3, 1, 1, 1, 96),
    (2, 128, 8, 8, 96, 3, 1, 1, 1, None),
]


@pytest.mark.parametrize("geom", GEOMETRIES, ids=lambda g: "x".join(str(e) for e in g))
@pytest.mark.parametrize("tag,zp", [("bf16", False), ("f16", True)])
@pytest.mark.parametrize("with_bias", [True, False])
def test_qbits_conv2d_grid(geom, tag, zp, with_bias):
    b, cin, h, w, cout, kk, s, p, d, group = geom
    x = make_input(b, cin, h, w, tag, seed=cin + h)
    bias = make_bias(cout, tag, cin) if with_bias else None
    y, wdeq = run_qbits(x, cout, kk, kk, group, tag, zp, bias, (s, s), (p, p), (d, d), seed=cout)
    assert N.load().qb200_last_kernel_family() == 5
    check_conv(y, x, wdeq, bias, tag, (s, s), (p, p), (d, d), f"{geom} {tag} zp={zp}")


@pytest.mark.parametrize("tag", ["bf16", "f16"])
def test_qbits_conv2d_padding_border(tag):
    x = make_input(2, 32, 9, 10, tag, seed=3, border=300.0)
    bias = make_bias(64, tag, 3)
    for p, d in ((1, 1), (2, 2), (2, 1)):
        y, wdeq = run_qbits(x, 64, 3, 3, 96, tag, False, bias, (1, 1), (p, p), (d, d), seed=7)
        check_conv(y, x, wdeq, bias, tag, (1, 1), (p, p), (d, d), f"border p={p} d={d}")


def test_qbits_conv2d_large():
    # SD-1.5-like level: sampled rows against the oracle, every element against fp32 cuDNN
    x = make_input(2, 320, 32, 32, "bf16", seed=11)
    bias = make_bias(320, "bf16", 11)
    y, wdeq = run_qbits(x, 320, 3, 3, 96, "bf16", False, bias, (1, 1), (1, 1), (1, 1), seed=5)
    check_conv(y, x, wdeq, bias, "bf16", (1, 1), (1, 1), (1, 1), "sd-320")


def test_unbatched_input():
    x = make_input(1, 32, 9, 9, "bf16", seed=1)
    y4, wdeq = run_qbits(x, 64, 3, 3, 96, "bf16", False, None, (1, 1), (1, 1), (1, 1), seed=2)
    y3, _ = run_qbits(x[0], 64, 3, 3, 96, "bf16", False, None, (1, 1), (1, 1), (1, 1), seed=2)
    assert y3.shape == y4.shape[1:]
    assert torch.equal(y3, y4[0])


# ---------------------------------------------------------------------------------------------- 8-bit grid
def qbytes_weight(cout, cin, kh, kw, wtag, tag, seed):
    g = torch.Generator().manual_seed(seed)
    if wtag == "int8":
        w = torch.randint(-127, 128, (cout, cin, kh, kw), generator=g, dtype=torch.int8)
    else:
        w = (torch.randn(cout, cin, kh, kw, generator=g) * 2).to(WDT[wtag])
    scale = (torch.rand(cout, 1, 1, 1, generator=g) * 0.01 + 0.001).to(DT[tag])
    w, scale = w.to(DEV), scale.to(DEV)
    wdeq = (w.float() * scale.float()).to(DT[tag])  # rnd(scale * W): exact product, one rounding
    return w, scale, wdeq


@pytest.mark.parametrize("wtag", list(WDT))
@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("geom", [GEOMETRIES[0], GEOMETRIES[3], GEOMETRIES[5]], ids=["3x3", "stride2", "ktail"])
def test_qbytes_conv2d_grid(wtag, tag, geom):
    b, cin, h, w, cout, kk, s, p, d, _ = geom
    x = make_input(b, cin, h, w, tag, seed=cin)
    bias = make_bias(cout, tag, cout) if wtag != "e5m2" else None
    wq, scale, wdeq = qbytes_weight(cout, cin, kk, kk, wtag, tag, seed=h)
    y = torch.ops.quanto.qbytes_conv2d(x, wq, scale, bias, [s, s], [p, p], [d, d])
    assert N.load().qb200_last_kernel_family() == 5
    check_conv(y, x, wdeq, bias, tag, (s, s), (p, p), (d, d), f"{geom} {wtag} {tag}")


# ------------------------------------------------------------------------------------------ every instantiation
@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("tag", ["bf16", "f16"])
@pytest.mark.parametrize("kind", ["float", "zp", "int8", "e4m3fn", "e5m2", "e4m3fnuz"])
def test_every_instantiation(tile, tag, kind):
    # edge shape: M = 2 * 7 * 9 = 126 (tiles straddle the two images, the last one ragged), K = 288 (a 32-k tail),
    # Cout = 130 (a second, nearly empty N tile)
    b, cin, h, w, cout = 2, 32, 7, 9, 130
    x = make_input(b, cin, h, w, tag, seed=tile)
    bias = make_bias(cout, tag, tile)
    with N.test_override(N.OVR_CONV_TILE_M, tile):
        if kind in ("float", "zp"):
            y, wdeq = run_qbits(x, cout, 3, 3, 96, tag, kind == "zp", bias, (1, 1), (1, 1), (1, 1), seed=tile)
        else:
            wq, scale, wdeq = qbytes_weight(cout, cin, 3, 3, kind, tag, seed=tile)
            y = torch.ops.quanto.qbytes_conv2d(x, wq, scale, bias, [1, 1], [1, 1], [1, 1])
        assert N.load().qb200_last_kernel_family() == 5
    check_conv(y, x, wdeq, bias, tag, (1, 1), (1, 1), (1, 1), f"{kind} {tag} tile {tile}")


@pytest.mark.parametrize("tile", [64, 128])
@pytest.mark.parametrize("kind", ["int4", "int8"])
def test_more_tiles_than_sms(tile, kind):
    """ResNet-50's 56x56x64 level at batch 8 (Cout 192: two N tiles): M = 25088 gives 392 / 196 M tiles, several per
    CTA of the persistent grid, so every role walks from one tile to the next (gather rows, ring positions, the
    staging's stage sequence, the consumers' loop).  Rows sampled per 32-row band against the oracle, every element
    against fp32 cuDNN."""
    b, cin, h, w, cout = 8, 64, 56, 56, 192
    m = b * h * w
    assert -(-m // tile) * 2 > torch.cuda.get_device_properties(0).multi_processor_count
    x = make_input(b, cin, h, w, "bf16", seed=tile)
    bias = make_bias(cout, "bf16", tile)
    with N.test_override(N.OVR_CONV_TILE_M, tile):
        if kind == "int4":
            y, wdeq = run_qbits(x, cout, 3, 3, 96, "bf16", False, bias, (1, 1), (1, 1), (1, 1), seed=tile)
        else:
            wq, scale, wdeq = qbytes_weight(cout, cin, 3, 3, "int8", "bf16", seed=tile)
            y = torch.ops.quanto.qbytes_conv2d(x, wq, scale, bias, [1, 1], [1, 1], [1, 1])
        assert N.load().qb200_last_kernel_family() == 5
    check_conv(y, x, wdeq, bias, "bf16", (1, 1), (1, 1), (1, 1), f"{kind} tile {tile}")


def test_unaligned_weight_takes_the_composition():
    """A packed weight read in place at an offset that breaks the 16-byte alignment of the kernel's loads: the C ABI
    declines it and F.conv2d runs the composition instead of raising."""
    _, qc = frozen_conv(64, 64, 1, q.qint4)
    w = qc.weight
    packed = w._data._data
    buf = torch.empty(packed.numel() + 1, dtype=torch.uint8, device=DEV)
    shifted = buf[1:].view(packed.shape)
    shifted.copy_(packed)
    assert shifted.is_contiguous() and shifted.data_ptr() % 16 != 0
    w._data._data = shifted
    x = make_input(2, 64, 9, 9, "bf16", seed=12)
    with torch.no_grad():
        y = qc(x)
        ref = composition(qc, x)
    assert torch.equal(y, ref)


def test_kernel_declines():
    x = make_input(1, 40, 8, 8, "bf16", seed=0)  # K = 360: K % 16 != 0
    packed, scale, shift, _ = qbits_weight(64, 360, 360, "bf16", False, 0)
    with pytest.raises(N.UnsupportedConfiguration):
        torch.ops.quanto.qbits_conv2d(x, packed, scale, shift, None, [64, 40, 3, 3], 360, 4, [1, 1], [1, 1], [1, 1])
    x = make_input(1, 32, 8, 8, "bf16", seed=0)  # K = 288 with groups of 48
    packed, scale, shift, _ = qbits_weight(64, 288, 48, "bf16", False, 0)
    with pytest.raises(N.UnsupportedConfiguration):
        torch.ops.quanto.qbits_conv2d(x, packed, scale, shift, None, [64, 32, 3, 3], 48, 4, [1, 1], [1, 1], [1, 1])


# --------------------------------------------------------------------------------------------- QConv2d module
def frozen_conv(cin, cout, k, weights, dtype=torch.bfloat16, seed=0, activations=None, **kw):
    torch.manual_seed(seed)
    conv = torch.nn.Conv2d(cin, cout, k, **kw).to(dtype).to(DEV)
    qc = q.QConv2d.from_module(conv, weights=weights, activations=activations)
    qc.freeze()
    return conv, qc


def composition(qc, x):
    """What the reference runs: the dequantised weight through F.conv2d (padding_mode handled by _conv_forward)."""
    return torch.nn.Conv2d._conv_forward(qc, x, qc.weight.dequantize(), qc.bias)


def one_rounding(qc, x):
    """The same in fp32, rounded once: the arithmetic of the reference's QConv2d on the CPU (bias in the sum)."""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        w = qc.weight.dequantize().float()
        b = None if qc.bias is None else qc.bias.float()
        return torch.nn.Conv2d._conv_forward(qc, x.float(), w, b).to(x.dtype)
    finally:
        torch.backends.cudnn.allow_tf32 = prev


@pytest.mark.parametrize("weights", [q.qint4, q.qint8, q.qfloat8_e4m3fn])
def test_qconv2d_end_to_end(weights):
    # K = Cin * kh * kw = 64: a conv the routing rule (library_conv.NATIVE_MAX_K) sends to the kernel
    conv, qc = frozen_conv(64, 96, 1, weights, padding=1)
    assert isinstance(qc.weight, (WeightQBitsTensor, WeightQBytesTensor))
    x = make_input(2, 64, 13, 11, "bf16", seed=4)
    with torch.no_grad():
        y = qc(x)
        assert N.load().qb200_last_kernel_family() == 5
        ref = one_rounding(qc, x)
        comp = composition(qc, x)  # cuDNN, then the bias add: one more rounding
    rel = float((y.float() - ref.float()).norm() / ref.float().norm())
    assert rel < 1e-3, rel
    assert float((y.float() - comp.float()).norm() / comp.float().norm()) < 1e-2


def test_qconv2d_quantized_output():
    _, qc = frozen_conv(32, 64, 3, q.qint4, activations=q.qint8, padding=1)
    with torch.no_grad():
        y = qc(make_input(1, 32, 8, 8, "bf16", seed=5))
    assert isinstance(y, ActivationQBytesTensor)


@pytest.mark.parametrize("case", ["fp32", "groups2", "depthwise", "reflect", "unfrozen", "qactivation", "channels_last"])
def test_composition_routes(case):
    dtype = torch.float32 if case == "fp32" else torch.bfloat16
    kw = {"padding": 1}
    cin, cout = 32, 64
    if case == "groups2":
        kw["groups"] = 2
    if case == "depthwise":
        cin, cout, kw["groups"] = 32, 32, 32
    k = 3
    if case == "reflect":  # a shape the rule sends to the kernel (K = 64)
        kw["padding_mode"] = "reflect"
        cin, k = 64, 1
    torch.manual_seed(0)
    conv = torch.nn.Conv2d(cin, cout, k, **kw).to(dtype).to(DEV)
    qc = q.QConv2d.from_module(conv, weights=q.qint4)
    if case != "unfrozen":
        qc.freeze()
    x = make_input(2, cin, 9, 9, "bf16", seed=6).to(dtype)
    if case == "channels_last":
        x = x.to(memory_format=torch.channels_last)
    if case == "qactivation":
        x = q.quantize_activation(x, qtype=q.qint8, scale=(x.abs().max() / 127).to(dtype))
    if case == "unfrozen":  # training: the weight needs its graph
        y = qc(x).detach()
    with torch.no_grad():
        if case != "unfrozen":
            y = qc(x)
        w = qc.qweight.dequantize()
        xin = x.dequantize() if isinstance(x, ActivationQBytesTensor) else x
        ref = torch.nn.Conv2d._conv_forward(qc, xin, w, qc.bias)
    if case == "reflect":  # padded by F.pad, then the kernel with padding 0
        ref = one_rounding(qc, x)
        rel = float((y.float() - ref.float()).norm() / ref.float().norm())
        assert rel < 1e-3, rel
    else:
        assert torch.equal(y, ref)


def test_qconv2d_gradient():
    """The reference's gradient test: an unfrozen QConv2d's weight and bias gradients are those of F.conv2d of the
    dequantised weight (straight-through quantisation)."""
    torch.manual_seed(0)
    conv = torch.nn.Conv2d(32, 64, 3, padding=1).to(torch.bfloat16).to(DEV)
    qc = q.QConv2d.from_module(conv, weights=q.qint4)
    x = make_input(2, 32, 8, 8, "bf16", seed=8).requires_grad_(True)
    y = qc(x)
    g = torch.randn_like(y)
    y.backward(g)
    w = qc.qweight.dequantize().detach().requires_grad_(True)
    b = qc.bias.detach().clone().requires_grad_(True)
    x2 = x.detach().clone().requires_grad_(True)
    F.conv2d(x2, w, b, padding=1).backward(g)
    assert torch.allclose(qc.weight.grad.float(), w.grad.float(), rtol=1e-2, atol=1e-2)
    assert torch.allclose(qc.bias.grad.float(), b.grad.float(), rtol=1e-2, atol=1e-2)
    assert torch.allclose(x.grad.float(), x2.grad.float(), rtol=1e-2, atol=1e-2)


@pytest.mark.parametrize("weights", [q.qint4, q.qint8, q.qfloat8_e4m3fn])
@pytest.mark.parametrize("cin,k", [(32, 3), (8, 3), (64, 1)])  # group 96, per-axis (K = 72), per-axis (K = 64)
def test_4d_freeze_one_launch(weights, cin, k):
    """freeze() of a CUDA conv weight runs the one-launch quantizer on the [Cout, Cin * kh * kw] view; its bytes, scales
    and shifts (and their shapes) are those of the composition."""
    torch.manual_seed(1)
    conv = torch.nn.Conv2d(cin, 64, k).to(torch.bfloat16).to(DEV)
    qc = q.QConv2d.from_module(conv, weights=weights)
    with torch.no_grad():
        fused = qc._fused_qweight()
    assert fused is not None
    qc.freeze()
    opt = qc.optimizer
    if weights.bits == 8:
        scale = opt(conv.weight.detach(), qtype=weights, axis=0)
        comp = q.quantize_weight(conv.weight.detach(), qtype=weights, axis=0, scale=scale)
    else:
        scale, shift = opt(conv.weight.detach(), qtype=weights, axis=0, group_size=qc.weight_group_size)
        comp = q.quantize_weight(conv.weight.detach(), qtype=weights, axis=0, scale=scale, shift=shift,
                                 group_size=qc.weight_group_size)
    sd_f, sd_c = {}, {}
    fused.save_to_state_dict(sd_f, "", False)
    comp.save_to_state_dict(sd_c, "", False)
    assert sorted(sd_f) == sorted(sd_c)
    for key in sd_f:
        assert sd_f[key].shape == sd_c[key].shape, key
        assert sd_f[key].dtype == sd_c[key].dtype, key
        assert torch.equal(sd_f[key].view(torch.uint8), sd_c[key].view(torch.uint8)), key


@pytest.mark.parametrize("cin", [32, 8])  # group 96, per-axis (K = 72)
def test_4d_freeze_hqq(cin):
    """freeze() with the HQQ optimizer: the fused two-launch search on the [Cout, Cin * kh * kw] view of a grouped CUDA
    conv weight gives the bytes, scales and shifts (and shapes) of the composition on the CPU, the reference's
    arithmetic.  A per-axis conv weight keeps the composition: the reference's sums over the 4-D slices run in another
    order than over the rows the kernel reproduces."""
    torch.manual_seed(3)
    conv = torch.nn.Conv2d(cin, 64, 3).to(torch.bfloat16)
    qc_cpu = q.QConv2d.from_module(conv, weights=q.qint4, optimizer=q.HqqOptimizer())
    qc_gpu = q.QConv2d.from_module(torch.nn.Conv2d(cin, 64, 3).to(torch.bfloat16).to(DEV), weights=q.qint4,
                                   optimizer=q.HqqOptimizer())
    with torch.no_grad():
        qc_gpu.weight.copy_(conv.weight.to(DEV))
        fused = qc_gpu._fused_qweight()
    if qc_gpu.weight_group_size is None:
        assert fused is None
        return
    assert fused is not None
    qc_cpu.freeze()
    sd_f, sd_c = {}, {}
    fused.save_to_state_dict(sd_f, "", False)
    qc_cpu.weight.save_to_state_dict(sd_c, "", False)
    assert sorted(sd_f) == sorted(sd_c)
    for key in sd_f:
        assert sd_f[key].shape == sd_c[key].shape, key
        assert sd_f[key].dtype == sd_c[key].dtype, key
        assert torch.equal(sd_f[key].cpu().view(torch.uint8), sd_c[key].view(torch.uint8)), key


def test_golden_reference_qconv2d():
    """Our QConv2d frozen on the GPU has the reference's state dict bit for bit, and its output is within 1e-3 in norm of
    the reference's CPU output."""
    gold = np.load(GOLDEN)
    qtypes = {"qint4": q.qint4, "qint8": q.qint8, "qfloat8_e4m3fn": q.qfloat8_e4m3fn}
    for i in range(int(gold["n"])):
        pre = f"c{i}_"
        cin, cout, k, s, p, d, group = (int(e) for e in gold[pre + "geom"])
        conv = torch.nn.Conv2d(cin, cout, k, stride=s, padding=p, dilation=d).to(torch.bfloat16)
        with torch.no_grad():
            conv.weight.copy_(bits_t(gold[pre + "w"], "bf16"))
            conv.bias.copy_(bits_t(gold[pre + "bias"], "bf16"))
        conv = conv.to(DEV)
        qc = q.QConv2d.from_module(conv, weights=qtypes[str(gold[pre + "wq"])])
        qc.freeze()
        assert (qc.weight_group_size or 0) == group
        sd = qc.state_dict()
        for key in gold.files:
            if key.startswith(pre + "sd_"):
                name = key[len(pre) + 3:]
                mine = torch_to_bits(sd[name])
                assert mine.shape == gold[key].shape, (i, name)
                assert np.array_equal(mine.view(np.uint8), np.ascontiguousarray(gold[key]).view(np.uint8)), (i, name)
        x = bits_t(gold[pre + "x"], "bf16")
        with torch.no_grad():  # the kernel, called directly: most fixture shapes are routed to the composition
            w = qc.weight
            if isinstance(w, WeightQBitsTensor):
                y = torch.ops.quanto.qbits_conv2d(x, w._data._data, w._scale, w._shift, qc.bias, list(w.shape),
                                                  w._group_size or cin * k * k, 4, [s, s], [p, p], [d, d])
            else:
                y = torch.ops.quanto.qbytes_conv2d(x, w._data, w._scale, qc.bias, [s, s], [p, p], [d, d])
            assert torch.equal(qc(x), y if cin * k * k <= 64 else composition(qc, x))
            y = y.float().cpu()
        ref = torch.from_numpy(O.to_f32(gold[pre + "y"], "bf16"))
        rel = float((y - ref).norm() / ref.norm())
        assert rel < 1e-3, (i, rel)


# ------------------------------------------------------------------------------------------------ torch.compile
class Stack(torch.nn.Module):
    def __init__(self, weights):
        super().__init__()
        torch.manual_seed(2)
        # K <= 64 everywhere (a 4x4 stride-2 patch embedding of 4 channels, then 1x1 convs): the kernel's route
        self.a = torch.nn.Conv2d(4, 64, 4, stride=2, padding=1)
        self.b = torch.nn.Conv2d(64, 64, 1)
        self.c = torch.nn.Conv2d(64, 32, 1)
        for name in ("a", "b", "c"):
            setattr(self, name, q.QConv2d.from_module(getattr(self, name).to(torch.bfloat16).to(DEV), weights=weights))
            getattr(self, name).freeze()

    def forward(self, x):
        return self.c(torch.relu(self.b(torch.relu(self.a(x)))))


@pytest.mark.parametrize("weights", [q.qint4, q.qint8])
@pytest.mark.parametrize("backend", ["aot_eager", "cudagraphs"])
def test_compile_conv_stack(weights, backend):
    torch._dynamo.reset()
    m = Stack(weights)
    x = make_input(2, 4, 16, 16, "bf16", seed=9)
    with torch.no_grad():
        ref = m(x)
        assert N.load().qb200_last_kernel_family() == 5
        opts = {"fullgraph": True} if backend == "aot_eager" else {"dynamic": False}
        cm = torch.compile(m, backend=backend, **opts)
        for _ in range(3):
            y = cm(x)
    assert torch.equal(y, ref)
