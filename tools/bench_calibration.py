"""Time one calibration batch three ways, taking turns in one process (CUDA events, median of rounds):

  native  `with Calibration(): model(x)`: one quanto::absmax_update_ launch per scale, no host synchronisation
  comp    the same mode forced onto the reference's ATen composition (absmax_scale + `_updated_scale`, whose
          torch.all(scale == 1) synchronises with the host once per scale)
  graph   the native step captured once in a CUDA graph and replayed (the input copied into the static buffer first)

    python tools/bench_calibration.py [--rounds 7] [--iters 10]

Models, bf16 on cuda:0 with qint8 frozen weights and qint8 activations, streamline on (the reference's default; after
the first batch every output hook is gone, so each step is the steady-state calibration forward):
  - a BERT-base-sized encoder layer over 16 x 512 tokens: pre-LN, QLinear q / k / v / o (768), one 768-wide attention
    head (bmm + softmax), QLinear 768 -> 3072 -> 768 with GELU, two QLayerNorms;
  - two Llama-3-8B decoder MLPs (gate / up 4096 -> 14336, down 14336 -> 4096, SiLU) at 1, 32 and 2048 tokens.
Every arm first runs one eager batch (kernel loading, streamline decisions).  "native host only" is the host time of the
native eager step without waiting for the device: where it equals the eager step time, the step is host-bound.  Prints
the card, power limit and max SM clock read in this run, and the command line.
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "optimum-quanto_b200"))

import quanto_b200 as q  # noqa: E402
from quanto_b200 import calibrate  # noqa: E402

DEV = torch.device("cuda:0")
BF16 = torch.bfloat16


class Encoder(torch.nn.Module):
    def __init__(self, d=768, ffn=3072):
        super().__init__()
        self.ln1 = torch.nn.LayerNorm(d)
        self.q = torch.nn.Linear(d, d)
        self.k = torch.nn.Linear(d, d)
        self.v = torch.nn.Linear(d, d)
        self.o = torch.nn.Linear(d, d)
        self.ln2 = torch.nn.LayerNorm(d)
        self.fc1 = torch.nn.Linear(d, ffn)
        self.fc2 = torch.nn.Linear(ffn, d)

    def forward(self, x):
        h = self.ln1(x)
        a = torch.softmax(torch.bmm(self.q(h), self.k(h).transpose(1, 2)), dim=-1)
        x = x + self.o(torch.bmm(a, self.v(h)))
        return x + self.fc2(torch.nn.functional.gelu(self.fc1(self.ln2(x))))


class LlamaMLP(torch.nn.Module):
    def __init__(self, d=4096, ffn=14336):
        super().__init__()
        self.gate_proj = torch.nn.Linear(d, ffn, bias=False)
        self.up_proj = torch.nn.Linear(d, ffn, bias=False)
        self.down_proj = torch.nn.Linear(ffn, d, bias=False)

    def forward(self, x):
        return x + self.down_proj(torch.nn.functional.silu(self.gate_proj(x)) * self.up_proj(x))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return f"{name}, power limit / max SM clock: {pl}"


def build(kind):
    torch.manual_seed(0)
    model = Encoder() if kind == "encoder" else torch.nn.Sequential(LlamaMLP(), LlamaMLP())
    model = model.to(DEV, BF16)
    q.quantize(model, weights=q.qint8, activations=q.qint8)
    q.freeze(model)
    return model


def timed(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters * 1e3  # us


def arms(kind, shape):
    """{arm: step()} over one model per arm, each warmed by one eager calibration batch."""
    x = torch.randn(shape, device=DEV, dtype=BF16)
    models = {name: build(kind) for name in ("native", "comp", "graph")}
    for name, model in models.items():
        calibrate._FORCE_COMPOSITION = name == "comp"
        with torch.no_grad(), q.Calibration():
            model(x)
    calibrate._FORCE_COMPOSITION = False

    def native():
        with torch.no_grad(), q.Calibration():
            models["native"](x)

    def comp():
        calibrate._FORCE_COMPOSITION = True
        try:
            with torch.no_grad(), q.Calibration():
                models["comp"](x)
        finally:
            calibrate._FORCE_COMPOSITION = False

    static = x.clone()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad(), torch.cuda.graph(graph), q.Calibration():
        models["graph"](static)

    def replay():
        static.copy_(x)
        graph.replay()

    return {"native": native, "comp": comp, "graph": replay}


def host_timed(fn, iters):
    """Host time of `iters` calls, without waiting for the device at the end: what the Python side of a step costs."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    t1 = time.perf_counter()
    torch.cuda.synchronize()
    return (t1 - t0) / iters * 1e6  # us


def spread(v):
    return f"{statistics.median(v):.0f} ({min(v):.0f}-{max(v):.0f})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    print(card())
    print(f"python tools/bench_calibration.py --rounds {args.rounds} --iters {args.iters}: us per step, median "
          "(min-max) over rounds")
    cases = [("BERT-base-sized encoder layer, 16x512 tokens", "encoder", (16, 512, 768))]
    cases += [(f"2 Llama-3-8B MLPs, {t} tokens", "llama", (t, 4096)) for t in (1, 32, 2048)]
    print("| model | native eager | composition eager | native CUDA graph | native host only | comp / native | "
          "native / graph |")
    print("|---|---|---|---|---|---|---|")
    for label, kind, shape in cases:
        fns = arms(kind, shape)
        for fn in fns.values():  # warm-up of every arm's steady state
            timed(fn, 2)
        times = {name: [] for name in list(fns) + ["host"]}
        for _ in range(args.rounds):
            for name, fn in fns.items():
                times[name].append(timed(fn, args.iters))
            times["host"].append(host_timed(fns["native"], args.iters))
        med = {name: statistics.median(v) for name, v in times.items()}
        print(f"| {label} | {spread(times['native'])} | {spread(times['comp'])} | {spread(times['graph'])} | "
              f"{spread(times['host'])} | {med['comp'] / med['native']:.2f}x | {med['native'] / med['graph']:.2f}x |",
              flush=True)
        del fns
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
