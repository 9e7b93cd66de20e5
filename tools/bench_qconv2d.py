"""Time the quantized conv2d three ways, taking turns in one process (CUDA events, median of rounds):

  native  quanto::qbits_conv2d / quanto::qbytes_conv2d called directly (implicit GEMM, csrc/conv_tc.cuh)
  ref     the reference's route: w.dequantize() + cuDNN F.conv2d (what qfallback runs), bias included
  cudnn   cuDNN on the unquantized bf16 weight

    python tools/bench_qconv2d.py [--rounds 7] [--iters 20] [--knockouts]

Each arm is timed twice.  "eager" = back-to-back calls from Python: what an eager model pays, host dispatch included
(a small conv measures the host, not the GPU).  "gpu" = the replay of a CUDA graph holding `--iters` calls: the GPU
work alone, what a captured or compiled model pays.  TFLOP/s = 2 * M * N * K over the native GPU time (M = B * Ho * Wo,
N = Cout, K = Cin * kh * kw).  The last column is the route a frozen QConv2d takes (library_conv.native_conv2d).

--knockouts loads the developer library (`make -C optimum-quanto_b200/csrc KNOCKOUTS=1`) and times the native kernel's
GPU time with the gather's loads removed (flag 8), the epilogue's stores removed (256) and both: what each costs.
Prints the card name, power limit and max SM clock read in this run first.
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "optimum-quanto_b200"))

import quanto_b200 as q  # noqa: E402

# (label, B, Cin, H, W, Cout, k, stride, padding, weights)
SHAPES = [
    ("sd15 64x64 320->320", 2, 320, 64, 64, 320, 3, 1, 1, "qint4"),
    ("sd15 32x32 640->640", 2, 640, 32, 32, 640, 3, 1, 1, "qint4"),
    ("sd15 16x16 1280->1280", 2, 1280, 16, 16, 1280, 3, 1, 1, "qint4"),
    ("sd15 1x1 shortcut 320->640 32x32", 2, 320, 32, 32, 640, 1, 1, 0, "qint4"),
    ("resnet50 56x56x64 b32", 32, 64, 56, 56, 64, 3, 1, 1, "qint4"),
    ("resnet50 28x28x128 b32", 32, 128, 28, 28, 128, 3, 1, 1, "qint4"),
    ("resnet50 14x14x256 b32", 32, 256, 14, 14, 256, 3, 1, 1, "qint4"),
    ("stride-2 64x64 320->320", 2, 320, 64, 64, 320, 3, 2, 1, "qint4"),
    ("sd15 32x32 640->640 qint8", 2, 640, 32, 32, 640, 3, 1, 1, "qint8"),
    ("resnet50 56x56x64 b8", 8, 64, 56, 56, 64, 3, 1, 1, "qint4"),
    ("resnet50 14x14x256 b1", 1, 256, 14, 14, 256, 3, 1, 1, "qint4"),
    ("1x1 64->256 56x56 b1", 1, 64, 56, 56, 256, 1, 1, 0, "qint4"),
    ("small 16x16 64->64 b1", 1, 64, 16, 16, 64, 3, 1, 1, "qint4"),
]


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


def build(label, b, cin, h, w, cout, k, s, p, wq, dev):
    torch.manual_seed(0)
    conv = torch.nn.Conv2d(cin, cout, k, stride=s, padding=p).to(torch.bfloat16).to(dev)
    qc = q.QConv2d.from_module(conv, weights=q.qtypes[wq])
    qc.freeze()
    wt = qc.weight
    x = torch.randn(b, cin, h, w, device=dev).to(torch.bfloat16)
    if wq == "qint4":
        g = wt._group_size or cin * k * k
        native = lambda: torch.ops.quanto.qbits_conv2d(x, wt._data._data, wt._scale, wt._shift, qc.bias,  # noqa: E731
                                                       list(wt.shape), g, 4, [s, s], [p, p], [1, 1])
    else:
        native = lambda: torch.ops.quanto.qbytes_conv2d(x, wt._data, wt._scale, qc.bias, [s, s], [p, p],  # noqa: E731
                                                        [1, 1])
    arms = {
        "native": native,
        "ref": lambda: torch.nn.functional.conv2d(x, wt.dequantize(), qc.bias, s, p),
        "cudnn": lambda: conv(x),
    }
    with torch.no_grad():  # inference: the route a frozen QConv2d takes
        out = q.library_conv.native_conv2d((x, wt, qc.bias, s, p), {}, type(wt) if wq == "qint4" else None,
                                           type(wt) if wq != "qint4" else None)
    routed = "ref" if out is None else "native"
    ho = (h + 2 * p - k) // s + 1
    wo = (w + 2 * p - k) // s + 1
    return arms, routed, 2.0 * b * ho * wo * cout * cin * k * k


def run_knockouts(args, dev):
    from quanto_b200 import _native as N

    lib = N.load()
    assert lib.qb200_developer_build() == 1, "the developer library was not loaded"
    modes = {"release": 0, "no gather loads": 8, "no stores": 256, "neither": 264}
    print(f"{'shape':36s} " + " ".join(f"{m:>16s}" for m in modes) + "   (native GPU ms per call)")
    for shape in SHAPES:
        arms, _, _ = build(*shape, dev)
        with torch.no_grad():
            replays = {}
            for m, flags in modes.items():
                lib.qb200_debug_set_flags(flags)  # read when the launch is recorded: baked into the graph
                replays[m] = graph_timed(arms["native"], args.iters)
            lib.qb200_debug_set_flags(0)
            times = {m: [] for m in modes}
            for _ in range(args.rounds):
                for m, r in replays.items():
                    times[m].append(r())
        print(f"{shape[0]:36s} " + " ".join(f"{median(times[m]):16.4f}" for m in modes))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--knockouts", action="store_true")
    args = ap.parse_args()
    torch.backends.cudnn.benchmark = True
    dev = torch.device("cuda:0")
    print(card())
    if args.knockouts:
        from quanto_b200 import _native as N

        N.use_developer_library()
        run_knockouts(args, dev)
        return
    print(f"{'':44s} {'---------- eager ms ----------':>32s} {'----------- gpu ms -----------':>32s}")
    print(f"{'shape':36s} {'GFLOP':>7s} {'native':>10s} {'ref':>10s} {'cudnn':>10s} {'native':>10s} {'ref':>10s} "
          f"{'cudnn':>10s} {'TF/s':>7s} {'gpu ref/nat':>11s} {'QConv2d runs':>13s}")
    for shape in SHAPES:
        arms, routed, flop = build(*shape, dev)
        with torch.no_grad():
            for fn in arms.values():
                fn()
            replays = {a: graph_timed(fn, args.iters) for a, fn in arms.items()}
            torch.cuda.synchronize()
            eager = {a: [] for a in arms}
            gpu = {a: [] for a in arms}
            for _ in range(args.rounds):
                for a, fn in arms.items():
                    eager[a].append(timed(fn, args.iters))
                    gpu[a].append(replays[a]())
        e = {a: median(t) for a, t in eager.items()}
        g = {a: median(t) for a, t in gpu.items()}
        print(f"{shape[0]:36s} {flop / 1e9:7.2f} {e['native']:10.4f} {e['ref']:10.4f} {e['cudnn']:10.4f} "
              f"{g['native']:10.4f} {g['ref']:10.4f} {g['cudnn']:10.4f} {flop / g['native'] / 1e9:7.1f} "
              f"{g['ref'] / g['native']:10.2f}x {routed:>13s}")


if __name__ == "__main__":
    main()
