"""Shared helpers for the GPU parity tests: bit-pattern <-> torch conversions and direct C-ABI callers."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "optimum-quanto_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from oracle import quanto_oracle as O  # noqa: E402

TORCH_DT = {"f32": torch.float32, "f16": torch.float16, "bf16": torch.bfloat16,
            "e4m3fn": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2, "e4m3fnuz": torch.float8_e4m3fnuz,
            "int8": torch.int8}
TAG_OF = {v: k for k, v in TORCH_DT.items()}


def bits_to_torch(arr: np.ndarray, tag: str, device="cuda") -> torch.Tensor:
    """Storage representation (oracle convention) -> torch tensor of the real dtype."""
    if tag == "f32":
        return torch.from_numpy(np.ascontiguousarray(arr, dtype=np.float32)).to(device)
    if tag in ("f16", "bf16"):
        t = torch.from_numpy(np.ascontiguousarray(arr).view(np.int16)).to(device)
        return t.view(TORCH_DT[tag])
    if tag in O.FP8_TAGS:
        t = torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8)).to(device)
        return t.view(TORCH_DT[tag])
    if tag == "int8":
        return torch.from_numpy(np.ascontiguousarray(arr).view(np.int8)).to(device)
    if tag == "uint8":
        return torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8)).to(device)
    raise ValueError(tag)


def torch_to_bits(t: torch.Tensor) -> np.ndarray:
    t = t.detach().contiguous().cpu()
    if t.dtype == torch.float32:
        return t.numpy()
    if t.dtype in (torch.float16, torch.bfloat16):
        return t.view(torch.int16).numpy().view(np.uint16)
    if t.dtype in (torch.float8_e4m3fn, torch.float8_e5m2, torch.float8_e4m3fnuz):
        return t.view(torch.uint8).numpy()
    return t.numpy()


def torch_to_f32(t: torch.Tensor) -> np.ndarray:
    return t.detach().to(torch.float32).cpu().numpy()


def native():
    from quanto_b200 import _native
    return _native


def cabi_unpack(packed: torch.Tensor, bits: int) -> torch.Tensor:
    n = native()
    lib = n.load()
    packed = packed.contiguous()
    out = torch.empty((packed.shape[0] * (8 // bits),) + tuple(packed.shape[1:]), dtype=torch.uint8, device=packed.device)
    n.check(lib.qb200_unpack(n.ptr(packed), n.ptr(out), packed.numel(), bits, n.stream_ptr(packed.device)), "unpack")
    return out


def cabi_quantize_symmetric(base, out_dtype, axis, scale):
    n = native()
    lib = n.load()
    base = base.contiguous()
    out = torch.empty(base.shape, dtype=out_dtype, device=base.device)
    if axis is None:
        outer, inner, mode = 1, base.numel(), 0
    elif axis == 0:
        outer, inner, mode = base.shape[0], base.numel() // base.shape[0], 1
    else:
        inner = base.shape[-1]
        outer, mode = base.numel() // inner, 2
    n.check(lib.qb200_quantize_symmetric(n.ptr(base), n.ptr(scale.contiguous()), n.ptr(out), outer, inner, mode,
                                         n.DTYPE_CODE[base.dtype], n.DTYPE_CODE[out_dtype], n.stream_ptr(base.device)),
            "quantize_symmetric")
    return out


def cabi_dequantize_qbits(packed, scale, shift, N, K, group, bits):
    n = native()
    lib = n.load()
    out = torch.empty((N, K), dtype=scale.dtype, device=packed.device)
    shift_is_int = 0 if shift.dtype.is_floating_point else 1
    n.check(lib.qb200_dequantize_qbits(n.ptr(packed), n.ptr(scale), n.ptr(shift), n.ptr(out), N, K, group, bits,
                                       n.DTYPE_CODE[scale.dtype], shift_is_int, n.stream_ptr(packed.device)),
            "dequantize_qbits")
    return out


def cabi_qbits_mm(x, packed, scale, shift, bias, N, K, group, use_workspace=True, bits=4):
    n = native()
    lib = n.load()
    x = x.contiguous()
    M = x.numel() // K
    out = torch.empty((M, N), dtype=x.dtype, device=x.device)
    shift_is_int = 0 if shift.dtype.is_floating_point else 1
    stream = n.stream_ptr(x.device)
    ws = n.workspace(x.device, stream, lib.qb200_qbits_mm_workspace_bytes(M, N, K)) if use_workspace else None
    n.check(lib.qb200_qbits_mm(n.ptr(x), n.ptr(packed), n.ptr(scale), n.ptr(shift), n.ptr(bias), n.ptr(out), M, N, K,
                               group, bits, n.DTYPE_CODE[x.dtype], shift_is_int, n.ptr(ws), 0 if ws is None else ws.numel(),
                               stream), "qbits_mm")
    return out


def cabi_qbytes_mm(a, w, scales, bias=None):
    n = native()
    lib = n.load()
    a = a.contiguous()
    w = w.contiguous()
    K = a.shape[-1]
    M = a.numel() // K
    N = w.shape[0]
    out = torch.empty((M, N), dtype=scales.dtype, device=a.device)
    n.check(lib.qb200_qbytes_mm(n.ptr(a), n.ptr(w), n.ptr(scales.contiguous()), n.ptr(bias), n.ptr(out), M, N, K,
                                n.DTYPE_CODE[a.dtype], n.DTYPE_CODE[w.dtype], n.DTYPE_CODE[scales.dtype],
                                n.stream_ptr(a.device)), "qbytes_mm")
    return out, lib.qb200_last_kernel_family()


def make_qbits_weights(N, K, group, tag, seed=0, zeropoint=False):
    """Synthetic canonical int4 weights (numpy): uniform nibbles, positive scales, shifts around 8*scale
    (the shape of what MaxOptimizer produces, reference bench/kernels/benchmark_w4a16.py:28-41)."""
    rng = np.random.default_rng(seed)
    rows = N * K // group
    q = rng.integers(0, 16, size=(rows, group), dtype=np.uint8)
    packed = O.pack_weights(q, 4)
    scale = O.from_f32((rng.random(rows, dtype=np.float32) * 0.01 + 0.002), tag)
    if zeropoint:
        shift = rng.integers(0, 16, size=rows, dtype=np.uint8)
    else:
        shift = O.from_f32(O.to_f32(scale, tag) * (7.0 + 2 * rng.random(rows, dtype=np.float32)), tag)
    return q, packed, scale, shift


def band_rows(M, seed, per_band=2):
    """`per_band` distinct rows of every 32-row band of [0, M): every tile / epilogue warp of any tiling is sampled."""
    rng = np.random.default_rng(seed)
    rows = []
    for b0 in range(0, M, 32):
        hi = min(32, M - b0)
        rows.extend((b0 + rng.choice(hi, size=min(per_band, hi), replace=False)).tolist())
    return np.array(sorted(rows), dtype=np.int64)


def check_full_against_device_fp32(y_gpu, x_t, w_t, bias_t, label):
    """All output elements against the fp32 product of the same operands (cuBLAS fp32, TF32 off), rounded the way the
    reference rounds.  Catches a misplaced / stale / skipped tile anywhere in the output."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        ref = torch.matmul(x_t.float(), w_t.float().t()).to(y_gpu.dtype)
        if bias_t is not None:
            ref = (ref + bias_t).to(y_gpu.dtype)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev
    d = (y_gpu.float() - ref.float())
    rel = float(d.norm() / ref.float().norm())
    assert rel < 1e-3, (label, rel)
    # per element: two results of the same exact sum rounded to the output dtype differ by at most one output ulp plus
    # the accumulation-order slack; 2^-6 relative + a small absolute floor is ~4 bf16 ulps
    tol = ref.float().abs() * 2.0 ** -6 + 2.0 ** -6 * ref.float().abs().mean()
    bad = int((d.abs() > tol).sum())
    assert bad == 0, (label, bad, float((d.abs() / tol).max()))
    return float((y_gpu == ref).float().mean())


def check_linear(y_gpu, x_bits, deq_bits, bias_bits, tag, label):
    """A linear of dequantised operands against the float64 oracle: per-element bound and norm error vs the
    reference-rounded result.  Returns the fraction of bit-identical outputs."""
    x = O.to_f32(x_bits, tag)
    w = O.to_f32(deq_bits, tag)
    bias = None if bias_bits is None else O.to_f32(bias_bits, tag)
    y64, y_ref, tol = O.linear_from_dequantized(x, w, bias, tag)
    y = torch_to_f32(y_gpu).astype(np.float64)
    # rounding allowance (half an output ulp per rounding step) + fp32 accumulation-order slack
    bound = 1.02 * tol + O.accumulate_allowance(x, w)
    err = np.abs(y - y64)
    assert np.all(err <= bound), (label, float(np.max(err / bound)), np.unravel_index(np.argmax(err / bound), err.shape))
    # versus the reference-rounded result: same numbers up to accumulation order => norm error << 1e-3
    yr = O.to_f32(y_ref, tag).astype(np.float64)
    rel = np.linalg.norm(y - yr) / max(np.linalg.norm(yr), 1e-30)
    assert rel < 1e-3, (label, rel)
    return float(np.mean(torch_to_bits(y_gpu) == y_ref))
