"""CPU oracle of one Calibration scale update (optimum/quanto/calibrate.py:31-34 `_updated_scale` applied to 37-61
`absmax_scale`).  TEST INFRASTRUCTURE ONLY; numpy, pinned to the reference by tests/golden/calibration.npz
(oracle/gen_golden_calibration.py).

Every ATen op of the reference rounds its float32 result to the scale dtype T:
    new   = rnd(max|x| / qmax)                                       (float32 true division)
    scale = new                                      if scale == 1
            rnd(rnd(scale * m) + rnd(new * om))      otherwise, m = float32(momentum), om = float32(1 - momentum)
with 1 - momentum evaluated in double, as Python does, before it becomes a float32 operand.  max propagates NaN.
"""
from __future__ import annotations

import numpy as np

from .quanto_oracle import from_f32, round_to, to_f32

TAGS = ("f32", "f16", "bf16")  # index = the dtype code stored in the fixture's metadata


def values(bits: np.ndarray, tag: str) -> np.ndarray:
    """The float32 values of T bit patterns (uint32 for f32, uint16 for f16 / bf16)."""
    if tag == "f32":
        return np.asarray(bits, np.uint32).view(np.float32)
    return to_f32(bits, tag)


def bits_of(x: np.ndarray, tag: str) -> np.ndarray:
    """The T bit patterns of float32 values already representable in T."""
    if tag == "f32":
        return np.asarray(x, np.float32).view(np.uint32)
    return np.asarray(from_f32(np.asarray(x, np.float32), tag)).view(np.uint16)


def absmax_update(scale: float, x: np.ndarray, qmax: float, momentum: float, tag: str) -> np.float32:
    """The scale (a float32 value representable in T) after one calibration step on the float32 values x."""
    with np.errstate(invalid="ignore", over="ignore"):
        a = np.abs(np.asarray(x, np.float32).reshape(-1))
        mx = np.float32(np.nan) if np.isnan(a).any() else a.max()
        new = round_to(np.array([mx / np.float32(qmax)], np.float32), tag)[0]
        scale = np.float32(scale)
        if scale == 1:
            return new
        m, om = np.float32(momentum), np.float32(1.0 - momentum)
        t = round_to(np.array([scale * m, new * om], np.float32), tag)
        return round_to(np.array([t[0] + t[1]], np.float32), tag)[0]
