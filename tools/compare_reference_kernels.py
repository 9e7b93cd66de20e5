"""Same-box comparison against the kernels the REFERENCE ITSELF dispatches to on this GPU (SURVEY 2.2 / BASELINE.md 5).

Runs the unmodified reference from oracle/_ref (python oracle/build_ref.py; its `quanto_cuda` extension -- AWQ v2, Marlin
FP8 -- pre-built for sm_90) in one process and this library in another, on the same Llama-3-8B shapes, CUDA-graph replay
over rotated weight copies (HBM-cold), CUDA events.  Reference routes (optimum/quanto/tensor/weights/qbits.py:97-138,
qbytes.py:122-143, library/qbytes_mm.py:73-88):
  fp16 x qint4 g128       -> AWQWeightQBitsTensor    -> quanto::gemm_f16i4_awq   (gemv rows < 8, else gemm; mma.sync)
  bf16 x qint4 g128       -> TinyGemmWeightQBitsTensor -> torch._weight_int4pack_mm
  fp16 x qfloat8_e4m3fn   -> MarlinF8QBytesTensor    -> quanto::gemm_f16f8_marlin
  int8 x int8             -> torch._int_mm + 2 elementwise passes

    python tools/compare_reference_kernels.py            # parent: runs both arms, prints a table, writes JSON
    python tools/compare_reference_kernels.py --arm ref|ours   (internal)
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")
SHAPES = [(14336, 4096), (4096, 14336), (4096, 4096)]  # (N, K)
MS = [1, 8, 32, 4096]


def graph_time_us(torch, fns, reps=10):
    """fns: one callable per rotated weight copy; returns us per call."""
    for f in fns:
        f()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for f in fns:
            f()
    for _ in range(2):
        g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * len(fns))


def arm_ref(part):
    sys.path.insert(0, REF)
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0")
    import torch
    import optimum.quanto as oq
    from optimum.quanto import AbsmaxOptimizer, MaxOptimizer, qfloat8_e4m3fn, qint4, qint8
    from optimum.quanto.tensor.weights import quantize_weight
    dev = torch.device("cuda")
    lin = torch.nn.functional.linear
    out = []

    def copies(N, K):
        return max(2, min(6, int(160e6 // (N * K // 2)) + 1))

    for N, K in SHAPES:
        for dtype, route in ((torch.float16, "awq_v2"), (torch.bfloat16, "tinygemm")):
            if route != part:
                continue
            ws = []
            for c in range(copies(N, K)):
                t = (torch.randn(N, K, device=dev) * 0.02).to(dtype)
                scale, shift = MaxOptimizer()(t, qtype=qint4, axis=0, group_size=128)
                ws.append(quantize_weight(t, qtype=qint4, axis=0, scale=scale, shift=shift, group_size=128, optimized=True))
            kind = type(ws[0]).__name__
            for M in reversed(MS):  # large M first: a faulting small-M kernel then costs only its own rows
                x = torch.randn(M, K, device=dev).to(dtype)
                try:
                    us = graph_time_us(torch, [lambda w=w: lin(x, w) for w in ws], reps=5 if M > 32 else 20)
                    out.append(dict(arm="reference", route=route, cls=kind, dtype=str(dtype), M=M, N=N, K=K, us=us))
                except Exception as e:  # noqa: BLE001
                    out.append(dict(arm="reference", route=route, cls=kind, dtype=str(dtype), M=M, N=N, K=K,
                                    error=f"{type(e).__name__}: {e}"[:200]))
                print(json.dumps(out[-1]), flush=True)
            del ws
            torch.cuda.empty_cache()
    N, K = 14336, 4096
    if part not in ("marlin_fp8", "int_mm"):
        return
    # fp16 x fp8 weights (Marlin FP8) and int8 x int8 (torch._int_mm route) at M = 4096 and decode sizes
    ws = []
    for c in range(2 if part == "marlin_fp8" else 0):
        t = (torch.randn(N, K, device=dev) * 0.02).to(torch.float16)
        scale = AbsmaxOptimizer()(t, qtype=qfloat8_e4m3fn, axis=0)
        ws.append(quantize_weight(t, qtype=qfloat8_e4m3fn, axis=0, scale=scale, optimized=True))
    for M in ((8, 4096) if part == "marlin_fp8" else ()):
        x = torch.randn(M, K, device=dev).to(torch.float16)
        try:
            us = graph_time_us(torch, [lambda w=w: lin(x, w) for w in ws], reps=5)
            out.append(dict(arm="reference", route="marlin_fp8", cls=type(ws[0]).__name__, dtype="fp16", M=M, N=N, K=K, us=us))
        except Exception as e:  # noqa: BLE001
            out.append(dict(arm="reference", route="marlin_fp8", M=M, N=N, K=K, error=f"{type(e).__name__}: {e}"[:200]))
        print(json.dumps(out[-1]), flush=True)
    if part != "int_mm":
        return
    a = torch.randint(-127, 127, (4096, K), dtype=torch.int8, device=dev)
    wi = torch.randint(-127, 127, (N, K), dtype=torch.int8, device=dev)
    sc = (torch.rand(N, 1, device=dev) / 1e3).to(torch.bfloat16)
    us = graph_time_us(torch, [lambda: torch.ops.quanto.qbytes_mm(a, wi, sc)] * 2, reps=5)
    out.append(dict(arm="reference", route="int_mm+epilogue", dtype="int8", M=4096, N=N, K=K, us=us))
    print(json.dumps(out[-1]), flush=True)


def arm_ours():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "optimum-quanto_b200"))
    import torch
    import quanto_b200 as q
    from bench import make_int4
    dev = torch.device("cuda")
    lin = torch.nn.functional.linear
    for N, K in SHAPES:
        for dtype in (torch.float16, torch.bfloat16):
            n_copies = max(2, min(6, int(160e6 // (N * K // 2)) + 1))
            ws = [make_int4(N, K, dev, seed=c, dtype=dtype) for c in range(n_copies)]
            for M in MS:
                x = torch.randn(M, K, device=dev).to(dtype)
                us = graph_time_us(torch, [lambda w=w: lin(x, w) for w in ws], reps=5 if M > 32 else 20)
                print(json.dumps(dict(arm="ours", route="qbits_mm", dtype=str(dtype), M=M, N=N, K=K, us=us)), flush=True)
    N, K = 14336, 4096
    g = torch.Generator(device=dev).manual_seed(1)
    for M in (8, 4096):
        x = torch.randn(M, K, device=dev).to(torch.float16)
        ws = []
        for c in range(2):
            wd = (torch.randn(N, K, device=dev, generator=g) * 2).to(torch.float8_e4m3fn)
            sc = (torch.rand(N, 1, device=dev, generator=g) / 1e2).to(torch.float16)
            ws.append(q.WeightQBytesTensor(q.qfloat8_e4m3fn, 0, wd.size(), wd.stride(), wd, sc, None))
        us = graph_time_us(torch, [lambda w=w: lin(x, w) for w in ws], reps=5)
        print(json.dumps(dict(arm="ours", route="qbytes_mm fp16 x fp8", dtype="fp16", M=M, N=N, K=K, us=us)), flush=True)
    a = torch.randint(-127, 127, (4096, K), dtype=torch.int8, device=dev)
    wi = torch.randint(-127, 127, (N, K), dtype=torch.int8, device=dev)
    sc = (torch.rand(N, 1, device=dev) / 1e3).to(torch.bfloat16)
    us = graph_time_us(torch, [lambda: torch.ops.quanto.qbytes_mm(a, wi, sc)] * 2, reps=5)
    print(json.dumps(dict(arm="ours", route="qbytes_mm int8", dtype="int8", M=4096, N=N, K=K, us=us)), flush=True)


def main():
    if "--arm" in sys.argv:
        arm = sys.argv[sys.argv.index("--arm") + 1]
        return arm_ours() if arm == "ours" else arm_ref(arm)
    rows = []
    # every reference kernel family in its own process: a kernel that faults on this GPU takes only its own rows with it
    for arm in ("awq_v2", "tinygemm", "marlin_fp8", "int_mm", "ours"):
        if arm != "ours" and not os.path.isdir(os.path.join(REF, "optimum")):
            print("oracle/_ref missing: reference arm skipped")
            continue
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--arm", arm], capture_output=True, text=True,
                           timeout=600)
        for line in r.stdout.splitlines():
            if line.startswith("{"):
                rows.append(json.loads(line))
        if r.returncode != 0:
            print(f"arm {arm} rc={r.returncode}: {r.stderr[-1500:]}")
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "compare_reference_kernels.json"), "w") as f:
        json.dump(rows, f, indent=1)
    for r in rows:
        flops = 2.0 * r["M"] * r["N"] * r["K"]
        if "us" in r:
            print(f"{r['arm']:9s} {r['route']:22s} {r.get('dtype', ''):15s} M={r['M']:5d} N={r['N']:5d} K={r['K']:5d} "
                  f"{r['us']:9.1f} us {flops / r['us'] / 1e6:8.1f} TF/s")
        else:
            print(f"{r['arm']:9s} {r['route']:22s} M={r['M']} N={r['N']} K={r['K']} ERROR {r['error']}")


if __name__ == "__main__":
    main()
