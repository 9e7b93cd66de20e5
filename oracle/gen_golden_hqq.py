"""Generate tests/golden/hqq.npz from the REAL reference's HqqOptimizer (huggingface/optimum-quanto, CPU path).

Run where a checkout of the reference is importable (the tests themselves never need it, they read the fixture):

    PYTHONPATH=<reference checkout> python oracle/gen_golden_hqq.py

A separate script and seed next to oracle/gen_golden.py (whose fixtures it leaves untouched); it reuses that script's
bit-pattern conventions.  The fixture pins oracle/hqq_oracle.py (tests/test_hqq_oracle.py) and is replayed against the
fused op (tests/test_gpu_hqq.py).
"""
import io
import os
import sys
from contextlib import redirect_stdout

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from gen_golden import OUT, TAG, bits  # noqa: E402  (imports optimum.quanto, registers torch.ops.quanto.*)
from optimum.quanto import HqqOptimizer, qint2, qint4  # noqa: E402
from optimum.quanto.tensor.optimizers import hqq_optimizer as hqq_module  # noqa: E402

ALL = torch.arange(0, 65536, dtype=torch.int32).to(torch.int16)  # every 16-bit pattern


def _recorded_errors(fn):
    """Run fn() and return what it returned plus every float() the optimizer took (start error, then one per
    iteration): the module's `float` is shadowed by a recorder, so the stored values are exact, not the 6-digit print."""
    seen = []

    def recording_float(x):
        v = float(x)
        seen.append(v)
        return v

    hqq_module.float = recording_float
    try:
        with redirect_stdout(io.StringIO()):
            out = fn()
    finally:
        del hqq_module.float
    return out, seen


def gen(g):
    cases = {}
    # pow(|x|, lp - 1) and shrink_lp_op on every pattern at the defaults (x = the pattern's index, not stored), other
    # lp_norm / beta on a random subset of patterns
    for dtype in (torch.bfloat16, torch.float16):
        tag = TAG[dtype]
        x = ALL.view(dtype)
        cases[f"pow_{tag}"] = bits(torch.pow(torch.abs(x), 0.7 - 1))
        for j, (lp, beta, full) in enumerate([(0.7, 10.0, True), (1.0, 10.0, False), (0.7, 10.0 * 1.01 ** 7, False),
                                              (0.7, 3.3, False), (1.0, 13.7, False), (0.8, 5.0, False)]):
            xs = x if full else x[torch.randperm(65536, generator=g)[:2048]]
            p = f"shrink_{tag}_{j}_"
            cases[p + "lp"] = np.float64(lp)
            cases[p + "beta"] = np.float64(beta)
            if not full:
                cases[p + "x"] = bits(xs)
            cases[p + "out"] = bits(hqq_module.shrink_lp_op(xs, beta, lp))
    # HqqOptimizer()(W, qtype, axis=0, group_size), zeropoint shifts as AffineOptimizer returns them
    cfgs = []
    for dtype in (torch.bfloat16, torch.float16):
        for qt in (qint4, qint2):
            for G, N in ((32, 20), (64, 12), (96, 14), (128, 20)):
                cfgs.append((dtype, qt, N, 384, G, False, {}, "normal"))
    cfgs += [
        (torch.bfloat16, qint4, 16, 256, 64, True, {}, "normal"),
        (torch.float16, qint2, 20, 192, 96, True, {}, "normal"),
        (torch.bfloat16, qint4, 12, 256, 128, False, dict(lp_norm=0.8, beta=5.0, kappa=1.05, iters=7), "normal"),
        (torch.float16, qint4, 12, 256, 64, False, dict(lp_norm=1.0, beta=20.0, kappa=1.1, iters=30), "normal"),
        (torch.bfloat16, qint4, 8, 256, 128, False, dict(iters=0), "normal"),
        (torch.bfloat16, qint4, 10, 256, 64, False, {}, "constant"),
        (torch.float16, qint2, 14, 128, 32, True, {}, "constant"),
    ]
    for idx, (dtype, qt, N, K, G, zp, kw, kind) in enumerate(cfgs):
        W = torch.randn(N, K, generator=g) * 0.02
        if kind == "constant":  # some all-zero groups and some constant ones
            Wg = W.view(-1, G)
            Wg[1::5] = 0.0
            Wg[3::7] = 0.0125
        W = W.to(dtype)
        opt = HqqOptimizer(verbose=True, **kw)
        (scale, shift), errs = _recorded_errors(lambda: opt(W, qtype=qt, axis=0, group_size=G, zeropoint=zp))
        p = f"h{idx}_"
        cases[p + "tag"] = np.array(TAG[dtype])
        cases[p + "bits"] = np.int64(qt.bits)
        cases[p + "shape"] = np.array([N, K, G], dtype=np.int64)
        cases[p + "zeropoint"] = np.int64(int(zp))
        cases[p + "params"] = np.array([opt.lp_norm, opt.beta, opt.kappa, opt.iters], dtype=np.float64)
        cases[p + "W"] = bits(W)
        cases[p + "scale"] = bits(scale)
        cases[p + "shift"] = bits(shift)
        cases[p + "errors"] = np.array(errs, dtype=np.float64)
    cases["n_hqq"] = np.int64(len(cfgs))
    # one QLinear freeze with the HQQ optimizer (qint4, group 128), kept in the canonical layout as gen_golden.py does
    from optimum.quanto.nn import QLinear

    lin = torch.nn.Linear(256, 32, bias=False).to(torch.bfloat16)
    with torch.no_grad():
        lin.weight.copy_((torch.randn(32, 256, generator=g) * 0.02).to(torch.bfloat16))
    q = QLinear.from_module(lin, weights=qint4, optimizer=HqqOptimizer())
    qw = q.qweight
    if type(qw).__name__ != "WeightQBitsTensor":
        qw = qw.weight_qbits_tensor()
    cases["qlinear_W"] = bits(lin.weight)
    cases["qlinear_group"] = np.int64(q.weight_group_size)
    cases["qlinear_packed"] = qw._data._data.numpy()
    cases["qlinear_scale"] = bits(qw._scale)
    cases["qlinear_shift"] = bits(qw._shift)
    np.savez_compressed(os.path.join(OUT, "hqq.npz"), **cases)


def main():
    torch.set_num_threads(1)  # deterministic accumulation order for the stored float results
    gen(torch.Generator().manual_seed(20261019))
    print("wrote", os.path.normpath(os.path.join(OUT, "hqq.npz")))
    return 0


if __name__ == "__main__":
    sys.exit(main())
