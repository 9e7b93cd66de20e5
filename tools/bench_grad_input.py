#!/usr/bin/env python
"""Times the input gradient of the quantized linear: the native kernel (qb200_qbits_mm_grad_input /
qb200_qbytes_mm_grad_input) against the composition it replaces (dequantise the weight to a dense [N, K] copy, then
torch.matmul), with CUDA events.

    python tools/bench_grad_input.py [--rounds 5] [--iters 10] [--out FILE]

For each shape both routes are warmed up, then take turns, `--iters` launches each, for `--rounds` rounds (clock and
neighbour drift hit both alike); the medians are reported.  The two outputs are compared against the parity bound
|native - composition| <= ulp + 2 * 2^-22 sqrt(N) (|gO| @ |Wd|) (each is within half an ulp plus the accumulation slack
of the exact product).  The card's name, power limit and SM clocks are read with an `nvidia-smi --query-gpu` query in the
same run (no setting is changed).  One JSON line per shape, and a summary table, go to stdout and to `--out`.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "optimum-quanto_b200"))

from quanto_b200 import _native as N  # noqa: E402

GROUP = 128
SHAPES_NK = [(14336, 4096), (4096, 14336), (4096, 4096), (1024, 4096)]
MS = [16, 128, 512, 2048, 4096]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock, max_clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "sm_clock": clock, "max_sm_clock": max_clock}


def int4_case(n, k, dtype, gen):
    lib = N.load()
    packed = torch.randint(0, 256, (n // 2, k), dtype=torch.uint8, device="cuda", generator=gen)
    scale = (torch.rand(n * k // GROUP, device="cuda", generator=gen) * 0.01 + 0.002).to(dtype)
    shift = (scale.float() * 8).to(dtype)
    code = N.DTYPE_CODE[dtype]

    def native(gO, out):
        N.check(lib.qb200_qbits_mm_grad_input(N.ptr(gO), N.ptr(packed), N.ptr(scale), N.ptr(shift), N.ptr(out),
                                              gO.shape[0], n, k, GROUP, code, 0, N.stream_ptr(gO.device)), "grad")

    def dequant():
        w = torch.empty((n, k), dtype=dtype, device="cuda")
        N.check(lib.qb200_dequantize_qbits(N.ptr(packed), N.ptr(scale), N.ptr(shift), N.ptr(w), n, k, GROUP, 4, code, 0,
                                           N.stream_ptr(w.device)), "dequantize")
        return w

    return native, dequant


def int8_case(n, k, dtype, gen):
    lib = N.load()
    w8 = torch.randint(-127, 128, (n, k), dtype=torch.int8, device="cuda", generator=gen)
    scale = (torch.rand(n, 1, device="cuda", generator=gen) * 0.01 + 0.001).to(dtype)

    def native(gO, out):
        N.check(lib.qb200_qbytes_mm_grad_input(N.ptr(gO), N.ptr(w8), N.ptr(scale), N.ptr(out), gO.shape[0], n, k,
                                               N.I8, N.DTYPE_CODE[dtype], N.stream_ptr(gO.device)), "grad")

    def dequant():
        return scale * w8  # QBytesDequantizer: scale * data in the scale dtype

    return native, dequant


def time_ms(fn, iters):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_grad_input needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    info = card()
    print(json.dumps({"card": info}), flush=True)
    gen = torch.Generator(device="cuda").manual_seed(0)
    dtype = torch.bfloat16
    rows = []
    cases = [("int4", n, k) for n, k in SHAPES_NK] + [("int8", 14336, 4096)]
    for kind, n, k in cases:
        native, dequant = (int4_case if kind == "int4" else int8_case)(n, k, dtype, gen)
        for m in MS:
            gO = torch.randn(m, n, device="cuda", generator=gen).to(dtype)
            out = torch.empty((m, k), dtype=dtype, device="cuda")
            composition = lambda: torch.matmul(gO, dequant())  # noqa: E731
            for _ in range(3):  # warm-up: module loads, cuBLAS heuristics
                native(gO, out)
                composition()
            torch.cuda.synchronize()
            t_nat, t_comp = [], []
            for _ in range(args.rounds):
                t_nat.append(time_ms(lambda: native(gO, out), args.iters))
                t_comp.append(time_ms(composition, args.iters))
            ref = composition()
            native(gO, out)
            wd = dequant().float()
            mag = torch.matmul(gO.float().abs(), wd.abs())
            ulp = torch.ldexp(torch.ones_like(mag), (torch.frexp(ref.float().abs().clamp_min(2.0 ** -126))[1] - 8))
            bound = ulp + 2 * 2.0 ** -22 * (n ** 0.5) * mag
            ratio = float(((out.float() - ref.float()).abs() / bound).max())
            nat, comp = statistics.median(t_nat), statistics.median(t_comp)
            flop = 2.0 * m * n * k
            row = {"kind": kind, "M": m, "N": n, "K": k, "native_ms": round(nat, 4), "composition_ms": round(comp, 4),
                   "speedup": round(comp / nat, 3), "native_tflops": round(flop / nat / 1e9, 1),
                   "max_err_over_bound": round(ratio, 3), "within_bound": ratio <= 1.0}
            rows.append(row)
            print(json.dumps(row), flush=True)
            del gO, out, ref, wd, mag, ulp, bound
    print(f"\n{info['name']}, power limit {info['power_limit']}, SM clock {info['sm_clock']} (max {info['max_sm_clock']})")
    print("| weights | N x K | M | native ms | dequantize + matmul ms | speed-up |")
    print("|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['kind']} | {r['N']} x {r['K']} | {r['M']} | {r['native_ms']:.3f} | {r['composition_ms']:.3f} | "
              f"{r['speedup']:.2f} |")
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"card": info, "rows": rows}, f, indent=1)
    if not all(r["within_bound"] for r in rows):
        raise SystemExit("native and composition outputs differ beyond the parity bound")


if __name__ == "__main__":
    main()
