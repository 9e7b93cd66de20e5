"""CPU oracle of the quantized layer norm (the reference's QLayerNorm, optimum/quanto/nn/qlayernorm.py, followed by the
quantize_output hook, nn/qmodule.py:296-302).  TEST INFRASTRUCTURE ONLY; numpy float64, pinned to the reference by
tests/golden/qlayernorm.npz (oracle/gen_golden_qlayernorm.py).

Parity contract.  n = (x - mu) / sigma is the float64 normalized value of the dequantized input, sigma =
sqrt(var + eps).  An element is flagged when moving y = gamma * n + beta by
    +- EPS * (|gamma| * (1 + |n| + |mu| / sigma) + |beta|)
moves it across a rounding boundary of the chain (the rounding to T, or the code boundary after it).  The |mu| / sigma
term covers the rounding of an fp32 mean (and implementations that compute x * rstd - mu * rstd, as torch's CPU kernel
does); |beta| covers the rounding of the final fp32 multiply-add.  Unflagged elements must give the oracle's code;
flagged ones at most one code away, or a code inside the band where the band spans more than one (`within_band`).
"""
from __future__ import annotations

import numpy as np

from .attention_oracle import code_distance, decode  # noqa: F401 (re-exported)
from .quanto_oracle import quantize_symmetric, round_to, to_f32  # noqa: F401

EPS = 1e-5


def dequantize(codes: np.ndarray, q_tag: str, scale_f32: float, tag: str) -> np.ndarray:
    """QBytesTensor.dequantize (tensor/qbytes.py:23-31): rnd_tag(scale * payload), as float32 values."""
    return round_to(np.float32(scale_f32) * decode(codes, q_tag), tag)


def normalize(x: np.ndarray, eps: float):
    """(n, mu, sigma) in float64 over the last axis of the float32 values x (already representable in T)."""
    x = np.asarray(x, np.float64)
    mu = x.mean(axis=-1, keepdims=True)
    var = ((x - mu) ** 2).mean(axis=-1, keepdims=True)
    sigma = np.sqrt(var + eps)
    return (x - mu) / sigma, mu, sigma


def affine(x: np.ndarray, weight, bias, eps: float, eps_contract: float = EPS):
    """(y64, band): the float64 layer norm output and the half-width of its contract band."""
    n, mu, sigma = normalize(x, eps)
    g = np.ones(x.shape[-1]) if weight is None else np.asarray(weight, np.float64)
    b = np.zeros(x.shape[-1]) if bias is None else np.asarray(bias, np.float64)
    y = g * n + b
    band = eps_contract * (np.abs(g) * (1 + np.abs(n) + np.abs(mu) / sigma) + np.abs(b))
    return y, band


def qlayer_norm(x, tag: str, weight, bias, eps: float, out_scale_f32: float, q_tag: str, eps_contract: float = EPS,
                band_codes: bool = False):
    """quantize_symmetric(rnd_tag(layer_norm(x)), q_tag, out_scale) -> (codes, flags), and with `band_codes` also the
    codes of the two ends of the band.  x, weight, bias: float32 values representable in `tag`; out_scale as float32
    (an fp32 scale with a 16-bit tag divides by the fp32 value)."""
    y, band = affine(x, weight, bias, eps, eps_contract)
    s = np.float32(out_scale_f32)

    def quantize(v):
        with np.errstate(over="ignore"):
            return quantize_symmetric(round_to(v.astype(np.float32), tag), tag, q_tag, s)

    out, lo, hi = quantize(y), quantize(y - band), quantize(y + band)
    flags = (lo != out) | (hi != out)
    return (out, flags, lo, hi) if band_codes else (out, flags)


def within_band(codes, lo, hi, q_tag: str) -> np.ndarray:
    """Whether each code lies between the codes of the band's ends (inclusive).  Near zero the fp8 codes are denser than
    the band of a row with |mu| >> sigma (a constant row: sigma = sqrt(eps)), so a flagged element may be several codes
    from the oracle's and still inside the band."""
    return (code_distance(codes, lo, q_tag) + code_distance(codes, hi, q_tag)) == code_distance(lo, hi, q_tag)


def layer_norm(x, tag: str, weight, bias, eps: float, eps_contract: float = EPS):
    """rnd_tag(layer_norm(x)) as float32 values -> (y, flags)."""
    y, band = affine(x, weight, bias, eps, eps_contract)

    def rnd(v):
        with np.errstate(over="ignore"):
            return round_to(v.astype(np.float32), tag)

    out = rnd(y)
    flags = (rnd(y - band) != out) | (rnd(y + band) != out)
    return out, flags
