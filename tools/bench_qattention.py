"""Time the quantized-attention ops against the reference's compositions, in one process, taking turns, CUDA events.

    python tools/bench_qattention.py [--iters 50] [--out results/bench_qattention.json]

Arms per workload (qbytes_ops.py:175-186, 208-215):
  native     quanto::qbytes_bmm / quanto::qbytes_softmax
  reference  the reference's arithmetic: fp32 casts + fp32 bmm (TF32 off) + scale + cast; or dequantize + softmax +
             quantize_symmetric
  bf16       torch.bmm of the dequantized bf16 operands (what a user without quantized attention runs)
GB/s counts the bytes an op must move: int8 operands read once, the [Bt, M, N] output written once (bf16), or the codes
read and written once for softmax.  The HBM roofline is the data sheet's 3.35 TB/s (H100 SXM).
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "optimum-quanto_b200"))

import quanto_b200  # noqa: E402,F401

HBM = 3.35e12


def timed(fns, iters):
    """Mean ms of each callable, alternating them every iteration."""
    for f in fns.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    ev = {k: [] for k in fns}
    for _ in range(iters):
        for k, f in fns.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            f()
            e.record()
            ev[k].append((s, e))
    torch.cuda.synchronize()
    return {k: sum(s.elapsed_time(e) for s, e in v) / len(v) for k, v in ev.items()}


def bench_bmm(bt, m, k, n, layout, iters):
    dev = "cuda"
    a = torch.randint(-127, 128, (bt, m, k), dtype=torch.int8, device=dev)
    if layout == "k":
        b = torch.randint(-127, 128, (bt, n, k), dtype=torch.int8, device=dev).transpose(1, 2)
    else:
        b = torch.randint(-127, 128, (bt, k, n), dtype=torch.int8, device=dev)
    sa = torch.tensor(0.01, dtype=torch.bfloat16, device=dev)
    sb = torch.tensor(0.02, dtype=torch.bfloat16, device=dev)
    ad, bd = (sa * a), (sb * b)
    torch.backends.cuda.matmul.allow_tf32 = False
    arms = {
        "native": lambda: torch.ops.quanto.qbytes_bmm(a, b, sa, sb),
        "reference": lambda: (torch.bmm(a.to(torch.float32), b.to(torch.float32)) * (sa * sb).to(torch.float32)).to(
            torch.bfloat16),
        "bf16": lambda: torch.bmm(ad, bd),
    }
    assert torch.equal(arms["native"](), arms["reference"]()) or k > 1024
    ms = timed(arms, iters)
    out = {"op": "qbytes_bmm", "shape": [bt, m, k, n], "b_layout": layout, "ms": ms}
    nbytes = bt * m * k + bt * k * n + 2 * bt * m * n
    out["bytes"] = nbytes
    out["GBps"] = {kk: nbytes / (v * 1e-3) / 1e9 for kk, v in ms.items()}
    out["roofline_share"] = {kk: (nbytes / HBM) / (v * 1e-3) for kk, v in ms.items()}
    return out


def bench_softmax(bt, m, n, iters):
    dev = "cuda"
    x = torch.randint(-127, 128, (bt, m, n), dtype=torch.int8, device=dev)
    s = torch.tensor(0.05, dtype=torch.bfloat16, device=dev)
    os_ = torch.tensor(1 / 127, dtype=torch.bfloat16, device=dev)
    arms = {
        "native": lambda: torch.ops.quanto.qbytes_softmax(x, s, os_),
        "reference": lambda: torch.ops.quanto.quantize_symmetric(torch.softmax(s * x, dim=-1), torch.int8, None, os_),
    }
    ms = timed(arms, iters)
    nbytes = 2 * x.numel()
    return {"op": "qbytes_softmax", "shape": [bt, m, n], "ms": ms, "bytes": nbytes,
            "GBps": {k: nbytes / (v * 1e-3) / 1e9 for k, v in ms.items()},
            "roofline_share": {k: (nbytes / HBM) / (v * 1e-3) for k, v in ms.items()}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_qattention needs a GPU")
    props = torch.cuda.get_device_properties(0)
    res = {"device": props.name, "results": [
        bench_bmm(32, 2048, 128, 2048, "k", args.iters),
        bench_bmm(32, 2048, 128, 2048, "n", args.iters),
        bench_bmm(256, 512, 64, 512, "k", args.iters),
        bench_bmm(32, 2048, 2048, 128, "n", args.iters),  # probs @ v, v N-contiguous
        bench_softmax(32, 2048, 2048, args.iters),
    ]}
    for r in res["results"]:
        print(json.dumps(r))
    if args.out:
        os.makedirs(os.path.dirname(args.out), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
