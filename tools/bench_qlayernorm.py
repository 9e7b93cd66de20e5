"""Time the quantized layer norm three ways, taking turns in one process (CUDA events, median of rounds):

  native  quanto::qbytes_layer_norm: bf16 floats or int8 codes in, int8 codes out, one launch
  comp    the reference's composition: (dequantize for codes in) + F.layer_norm + quanto::quantize_symmetric
  floor   F.layer_norm alone on the bf16 floats (no quantisation at all)

    python tools/bench_qlayernorm.py [--rounds 7] [--iters 20]

Each arm is timed twice.  "eager" = back-to-back calls from Python: what an eager model pays, host dispatch included.
"gpu" = the replay of a CUDA graph holding `--iters` calls: the GPU work alone.  GB/s = (input + output + gamma / beta
bytes) over the native GPU time, against the 3.35 TB/s of the H100 SXM data sheet.  Prints the card name, power limit
and max SM clock read in this run first.
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "optimum-quanto_b200"))

import quanto_b200  # noqa: E402,F401

# (label, rows, H)
SHAPES = [
    ("BERT-base 16x512x768", 16 * 512, 768),
    ("ViT-L 64x257x1024", 64 * 257, 1024),
    ("4096x4096", 4096, 4096),
    ("decode 1x4096", 1, 4096),
    ("decode 8x4096", 8, 4096),
    ("decode 32x4096", 32, 4096),
    ("2048x8192", 2048, 8192),
    ("1024x16384", 1024, 16384),
]
PEAK_GBS = 3350.0


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return f"{name}, power limit / max SM clock: {pl}"


def timed(fn, iters):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / iters


def graph_timed(fn, iters):
    """GPU time of one call: a CUDA graph of `iters` calls, replayed once (after one warm-up replay)."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(iters):
            fn()
    graph.replay()
    return lambda: timed(graph.replay, 1) / iters


def median(t):
    return sorted(t)[len(t) // 2]


def arms(rows, h, src, dev):
    torch.manual_seed(0)
    dt = torch.bfloat16
    x = torch.randn(rows, h, device=dev, dtype=dt)
    w = torch.randn(h, device=dev, dtype=dt)
    b = torch.randn(h, device=dev, dtype=dt)
    s_out = torch.tensor(0.05, device=dev, dtype=dt)
    ln = torch.nn.functional.layer_norm
    qs = torch.ops.quanto.quantize_symmetric
    if src == "codes":
        s_in = torch.tensor(0.03, device=dev, dtype=dt)
        codes = qs(x, torch.int8, None, s_in)
        native = lambda: torch.ops.quanto.qbytes_layer_norm(codes, s_in, [h], w, b, 1e-5, s_out, torch.int8)  # noqa
        comp = lambda: qs(ln(s_in * codes, [h], w, b, 1e-5), torch.int8, None, s_out)  # noqa: E731
        in_bytes = rows * h
    else:
        native = lambda: torch.ops.quanto.qbytes_layer_norm(x, None, [h], w, b, 1e-5, s_out, torch.int8)  # noqa
        comp = lambda: qs(ln(x, [h], w, b, 1e-5), torch.int8, None, s_out)  # noqa: E731
        in_bytes = 2 * rows * h
    floor = lambda: ln(x, [h], w, b, 1e-5)  # noqa: E731
    nbytes = in_bytes + rows * h + 2 * 2 * h
    return {"native": native, "comp": comp, "floor": floor}, nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    print(card())
    print(f"{'shape':24s} {'in':5s} | {'eager us: native':>16s} {'comp':>8s} {'floor':>8s} | {'gpu us: native':>14s} "
          f"{'comp':>8s} {'floor':>8s} | {'GB/s':>6s} {'of peak':>7s} {'gpu comp/native':>15s}")
    for label, rows, h in SHAPES:
        for src in ("float", "codes"):
            fns, nbytes = arms(rows, h, src, dev)
            graphs = {k: graph_timed(f, args.iters) for k, f in fns.items()}
            for f in fns.values():
                timed(f, 3)
            eager = {k: [] for k in fns}
            gpu = {k: [] for k in fns}
            for _ in range(args.rounds):
                for k in fns:  # the arms take turns
                    eager[k].append(timed(fns[k], args.iters) * 1e3)
                    gpu[k].append(graphs[k]() * 1e3)
            e = {k: median(v) for k, v in eager.items()}
            g = {k: median(v) for k, v in gpu.items()}
            gbs = nbytes / (g["native"] * 1e-6) / 1e9
            print(f"{label:24s} {src:5s} | {e['native']:16.1f} {e['comp']:8.1f} {e['floor']:8.1f} | "
                  f"{g['native']:14.2f} {g['comp']:8.2f} {g['floor']:8.2f} | {gbs:6.0f} {gbs / PEAK_GBS:7.1%} "
                  f"{g['comp'] / g['native']:15.2f}x", flush=True)


if __name__ == "__main__":
    main()
