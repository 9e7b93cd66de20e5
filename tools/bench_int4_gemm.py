#!/usr/bin/env python
"""Times the int4 linear (qb200_qbits_mm) through the C-ABI of one or more builds of the library, with CUDA events.

    python tools/bench_int4_gemm.py --lib parent=build/parent/libquanto_b200.so --lib new=optimum-quanto_b200/quanto_b200/lib/libquanto_b200.so [--out FILE]

Every `--lib NAME=PATH` is loaded into the same process.  For each shape the libraries take turns, one launch set each,
for `--rounds` rounds, so that clock and neighbour drift hit all of them alike; the JSON line reports each library's
median and best time per launch and the achieved TFLOP/s.  The card's name, power limit and maximum SM clock are read
with an `nvidia-smi --query-gpu` query (no setting is changed).
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess

import torch

# (label, M, N, K, dtype, zero-point)
SHAPES = [("gate_up_bf16", 4096, 14336, 4096, torch.bfloat16, False),
          ("down_bf16", 4096, 4096, 14336, torch.bfloat16, False),
          ("gate_up_f16_zp", 4096, 14336, 4096, torch.float16, True)] + \
         [(f"m{m}_bf16", m, 14336, 4096, torch.bfloat16, False) for m in (32, 64, 128, 256, 300, 512, 1024, 2048)] + \
         [(f"m{m}_n{n}_bf16", m, n, 4096, torch.bfloat16, False) for m, n in ((100, 128256), (128, 128256), (128, 33792),
                                                                               (4097, 14336))]
GROUP = 128
DT = {torch.float16: 1, torch.bfloat16: 2}


def load(path):
    lib = ctypes.CDLL(os.path.abspath(path))
    vp, i64, i32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
    lib.qb200_qbits_mm.argtypes = [vp, vp, vp, vp, vp, vp, i64, i64, i64, i32, i32, i32, i32, vp, i64, vp]
    lib.qb200_qbits_mm_workspace_bytes.argtypes = [i64, i64, i64]
    lib.qb200_qbits_mm_workspace_bytes.restype = i64
    lib.qb200_last_error.restype = ctypes.c_char_p
    return lib


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = [s.strip() for s in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def weights(N, K, dtype, zp, copies, gen):
    """`copies` independent canonical int4 weights ([N/2, K] packed bytes, [N, K/G] scale and shift)."""
    out = []
    for _ in range(copies):
        packed = torch.randint(0, 256, (N // 2, K), dtype=torch.uint8, device="cuda", generator=gen)
        scale = (torch.rand(N, K // GROUP, device="cuda", generator=gen) * 0.01 + 0.002).to(dtype)
        if zp:
            shift = torch.randint(0, 16, (N, K // GROUP), dtype=torch.uint8, device="cuda", generator=gen)
        else:
            shift = (scale.float() * 8).to(dtype)
        out.append((packed, scale, shift))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", required=True, help="NAME=PATH of a libquanto_b200.so build (repeatable)")
    ap.add_argument("--launches", type=int, default=10, help="launches per timed set")
    ap.add_argument("--rounds", type=int, default=6, help="timed sets per library and shape (taken in turns)")
    ap.add_argument("--only", default=None, help="comma-separated shape labels")
    ap.add_argument("--out", default=None, help="also write the JSON to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_int4_gemm needs a GPU"
    libs = []
    for spec in args.lib:
        name, path = spec.split("=", 1) if "=" in spec else (os.path.basename(os.path.dirname(spec)), spec)
        libs.append((name, load(path)))
    stream = torch.cuda.current_stream().cuda_stream
    gen = torch.Generator(device="cuda").manual_seed(0)
    result = {"card": card(), "launches_per_set": args.launches, "rounds": args.rounds, "shapes": {}}
    for label, M, N, K, dtype, zp in SHAPES:
        if args.only and label not in args.only.split(","):
            continue
        # enough weight copies that a launch does not find its weight in L2 (50 MB) from the launch before
        wbytes = N * K // 2
        ws = weights(N, K, dtype, zp, max(1, min(4, -(-96 * 2**20 // wbytes))), gen)
        x = torch.randn(M, K, device="cuda", generator=gen).to(dtype)
        outs = {name: torch.empty(M, N, dtype=dtype, device="cuda") for name, _ in libs}
        wsp = {}
        for name, lib in libs:
            nb = lib.qb200_qbits_mm_workspace_bytes(M, N, K)
            wsp[name] = (torch.zeros(max(nb, 1), dtype=torch.uint8, device="cuda"), nb)

        def launch(name, lib, i):
            packed, scale, shift = ws[i % len(ws)]
            buf, nb = wsp[name]
            rc = lib.qb200_qbits_mm(x.data_ptr(), packed.data_ptr(), scale.data_ptr(), shift.data_ptr(), None,
                                    outs[name].data_ptr(), M, N, K, GROUP, 4, DT[dtype], 1 if zp else 0,
                                    buf.data_ptr() if nb else None, nb, stream)
            if rc != 0:
                raise RuntimeError(f"{name}: qbits_mm failed: {lib.qb200_last_error().decode()}")

        for name, lib in libs:  # warm-up: module load, smem opt-in, clocks
            for i in range(3 * args.launches):
                launch(name, lib, i)
        torch.cuda.synchronize()
        times = {name: [] for name, _ in libs}
        for _ in range(args.rounds):
            for name, lib in libs:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(args.launches):
                    launch(name, lib, i)
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / args.launches)
        ref = outs[libs[0][0]]
        row = {"M": M, "N": N, "K": K, "dtype": str(dtype).replace("torch.", ""), "zero_point": zp}
        for name, _ in libs:
            med = statistics.median(times[name])
            row[name] = {"ms_median": round(med, 4), "ms_best": round(min(times[name]), 4),
                         "ms_worst": round(max(times[name]), 4), "tflops_median": round(2 * M * N * K / med / 1e9, 1),
                         "bit_identical_to_" + libs[0][0]: bool(torch.equal(outs[name], ref))}
        result["shapes"][label] = row
        print(json.dumps({label: row}), flush=True)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
