#!/usr/bin/env python
"""One Llama-3-8B decode step of qint4 linears, eager against torch.compile against a hand-captured CUDA graph.

    python tools/bench_compile.py [--batches 1 8 32] [--steps 50] [--rounds 5] [--out FILE]

The step runs the 224 linears of the 32 layers (q, k, v, o, gate, up, down; K = 4096, down K = 14336) as frozen
`QLinear` modules whose packed weights, scales and shifts are random and generated on the device.  Three arms run
the same modules in one process:
  eager       the step called directly (one Python __torch_function__ / autograd / op dispatch per linear);
  compiled    `torch.compile(step, backend="cudagraphs", fullgraph=True, dynamic=False)`, replayed by cudagraph trees;
  captured    a `torch.cuda.CUDAGraph` captured by hand around the step, as bench.py does.
All three outputs (the last hidden state and every layer's k and v) must be `torch.equal`, else the tool fails.  After
a warm-up, the arms take turns for `--rounds` rounds of `--steps` steps each, timed with CUDA events; the median per
arm is reported as ms per step and tokens/s (batch / step time).  The card's name, power limit and SM clocks are read
with an `nvidia-smi --query-gpu` query in the same run (no setting is changed).
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "optimum-quanto_b200"))

import quanto_b200 as q  # noqa: E402
from quanto_b200.tensor import PackedTensor, WeightQBitsTensor  # noqa: E402

HIDDEN, KV, FFN, LAYERS, GROUP = 4096, 1024, 14336, 32, 128
PROJ = [("q", HIDDEN, HIDDEN), ("k", KV, HIDDEN), ("v", KV, HIDDEN), ("o", HIDDEN, HIDDEN), ("gate", FFN, HIDDEN),
        ("up", FFN, HIDDEN), ("down", HIDDEN, FFN)]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    name, power, clock, max_clock = [s.strip() for s in out.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "sm_clock": clock, "max_sm_clock": max_clock}


def random_qlinear(n, k, gen):
    """A frozen qint4 QLinear (group 128, float shift) with random packed weights, centred so outputs stay O(1)."""
    lin = q.QLinear(k, n, bias=False, dtype=torch.bfloat16, device="meta", weights=q.qint4)
    rows = n * k // GROUP
    packed = torch.randint(0, 256, (rows // 2, GROUP), dtype=torch.uint8, device="cuda", generator=gen)
    scale = ((torch.rand(rows, 1, device="cuda", generator=gen) + 0.5) / (4.6 * math.sqrt(k))).to(torch.bfloat16)
    shift = (scale.float() * 7.5).to(torch.bfloat16)  # value = scale * q - shift, q in [0, 15]
    data = PackedTensor(packed, 4, torch.Size([rows, GROUP]), (GROUP, 1))
    w = WeightQBitsTensor(q.qint4, 0, GROUP, torch.Size([n, k]), (k, 1), data, scale, shift)
    lin = lin.to_empty(device="cuda")
    lin.weight = torch.nn.Parameter(w, requires_grad=False)
    return lin


class DecodeLinears(torch.nn.Module):
    """The 224 linears of one decode step; attention is left out, a max-norm stands in for RMSNorm, the MLP keeps its
    gate * up product."""

    def __init__(self, gen):
        super().__init__()
        self.layers = torch.nn.ModuleList(
            torch.nn.ModuleDict({name: random_qlinear(n, k, gen) for name, n, k in PROJ}) for _ in range(LAYERS))

    def forward(self, h):
        ks, vs = [], []
        for layer in self.layers:
            h = h / h.abs().amax(-1, keepdim=True)  # a cheap norm: keeps the gate * up product from growing per layer
            ks.append(layer["k"](h))
            vs.append(layer["v"](h))
            h = layer["o"](layer["q"](h))
            h = layer["down"](layer["gate"](h) * layer["up"](h))
        return (h, *ks, *vs)


def timed(fn, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8, 32])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_compile.py needs a CUDA device")
    gen = torch.Generator(device="cuda").manual_seed(0)
    model = DecodeLinears(gen)
    compiled = torch.compile(model, backend="cudagraphs", fullgraph=True, dynamic=False)  # one graph per batch
    info = card()
    rows = []
    with torch.no_grad():
        for batch in args.batches:
            x = torch.randn(batch, HIDDEN, dtype=torch.bfloat16, device="cuda", generator=gen)
            ref = model(x)
            for _ in range(3):  # cudagraph trees: warm-up, record, replay
                out_c = [t.clone() for t in compiled(x)]
            torch.cuda.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out_g = model(x)
            graph.replay()
            torch.cuda.synchronize()
            same = all(torch.equal(a, b) and torch.equal(a, c) for a, b, c in zip(ref, out_c, out_g))
            finite = bool(torch.isfinite(ref[0]).all())
            arms = {"eager": lambda: model(x), "compiled": lambda: compiled(x), "captured": graph.replay}
            for fn in arms.values():
                timed(fn, args.warmup)
            times = {name: [] for name in arms}
            for _ in range(args.rounds):
                for name, fn in arms.items():
                    times[name].append(timed(fn, args.steps))
            skips = dict(torch._dynamo.utils.counters["inductor"])  # cudagraph trees count the graphs they decline
            row = {"batch": batch, "identical": same, "finite": finite, "cudagraph_skips": skips.get("cudagraph_skips", 0)}
            for name, ts in times.items():
                ms = statistics.median(ts)
                row[name] = {"ms_per_step": round(ms, 4), "tokens_per_s": round(batch / ms * 1e3, 1),
                             "spread_ms": [round(min(ts), 4), round(max(ts), 4)]}
            row["card"] = info
            rows.append(row)
            print(json.dumps(row), flush=True)
            del graph, out_g
    print(f"\n{info['name']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}; "
          f"224 qint4 linears per step, median of {args.rounds} rounds x {args.steps} steps")
    print(f"{'batch':>5} | {'eager ms':>9} {'tok/s':>8} | {'compiled ms':>11} {'tok/s':>8} | {'captured ms':>11} "
          f"{'tok/s':>8} | identical")
    for r in rows:
        e, c, g = r["eager"], r["compiled"], r["captured"]
        print(f"{r['batch']:>5} | {e['ms_per_step']:>9.3f} {e['tokens_per_s']:>8.1f} | {c['ms_per_step']:>11.3f} "
              f"{c['tokens_per_s']:>8.1f} | {g['ms_per_step']:>11.3f} {g['tokens_per_s']:>8.1f} | {r['identical']}")
    if args.out:
        with open(args.out, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")
    if not all(r["identical"] and r["finite"] for r in rows):
        raise SystemExit("outputs differ between the arms (or are not finite)")


if __name__ == "__main__":
    main()
