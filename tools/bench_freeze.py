"""Developer micro-benchmark of the weight-freeze / calibration kernels (csrc/freeze.cu) and of the other HBM-bound
element kernels: CUDA events, rotated inputs larger than L2, achieved GB/s on the ALGORITHMIC bytes (DESIGN.md section 3)
next to the reference's own composition (ATen ops on the same GPU, optimum/quanto/nn/qmodule.py:245-266).

    python tools/bench_freeze.py > gpurun_out/freeze_bench.json
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "optimum-quanto_b200"))
import quanto_b200 as q  # noqa: E402
from quanto_b200.library import quantize_affine_any  # noqa: E402


def timeit(fn, iters=12, warmup=2, reps=5):
    """Seconds per call, device time: `iters` calls (rotated inputs) captured in one CUDA graph and replayed, so the
    Python / ctypes launch cost (15-25 us per call, more than several of these kernels take) is not in the number."""
    for i in range(warmup):
        fn(i)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for i in range(iters):
            fn(i)
    graph.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        graph.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (reps * iters) * 1e-3


def main():
    dev = "cuda"
    peaks_path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    hbm = json.load(open(peaks_path))["hbm_gbs"] if os.path.exists(peaks_path) else 6650.0
    res = {"hbm_peak_gbs": hbm}
    N, K, G = 14336, 4096, 128  # Llama-3-8B gate/up projection
    nrot = 3  # 3 x 117 MB of bf16 weights > 126 MB of L2
    ws = [(torch.randn(N, K, device=dev) * 0.02).to(torch.bfloat16) for _ in range(nrot)]
    rows = N * K // G

    if "--ncu" in sys.argv:  # a few launches of the kernels, for a profiler
        xs = torch.randn(4096, 4096, device=dev, dtype=torch.bfloat16)
        sc = torch.tensor(0.03, device=dev, dtype=torch.bfloat16)
        for i in range(3):
            torch.ops.quanto.quantize_qbits_max(ws[i % nrot], 4, G, False)
            torch.ops.quanto.quantize_symmetric(xs, torch.int8, None, sc)
            torch.ops.quanto.quantize_qbytes_absmax(ws[i % nrot], torch.int8)
        torch.cuda.synchronize()
        return

    def report(name, seconds, nbytes):
        res[name] = {"us": seconds * 1e6, "GBs": nbytes / seconds / 1e9, "frac_hbm": nbytes / seconds / 1e9 / hbm}

    # fused freeze, int4: read 2 B/weight, write 0.5 B/weight + scale/shift
    t = timeit(lambda i: torch.ops.quanto.quantize_qbits_max(ws[i % nrot], 4, G, False))
    report("quantize_qbits_max_bf16_int4", t, N * K * 2 + N * K // 2 + rows * 4)
    t = timeit(lambda i: torch.ops.quanto.quantize_qbits_max(ws[i % nrot], 4, G, True))
    report("quantize_qbits_max_bf16_int4_zeropoint", t, N * K * 2 + N * K // 2 + rows * 3)
    # the reference's composition on the same GPU: MaxOptimizer (ATen) + quantize_affine (ATen) + pack loop (ATen)
    opt = q.MaxOptimizer()

    def ref_freeze(i):
        w = ws[i % nrot]
        scale, shift = opt(w, qtype=q.qint4, axis=0, group_size=G)
        data = quantize_affine_any(w, 4, 0, G, scale, shift)
        r = data.shape[0] // 2
        return data[:r] | (data[r:] << 4)

    t = timeit(ref_freeze, iters=3, warmup=1, reps=3)
    report("reference_composition_aten_int4", t, N * K * 2 + N * K // 2 + rows * 4)
    # unfused kernels
    scale, shift = opt(ws[0], qtype=q.qint4, axis=0, group_size=G)
    t = timeit(lambda i: torch.ops.quanto.quantize_affine(ws[i % nrot], 4, 0, G, scale, shift))
    report("quantize_affine_bf16", t, N * K * 3 + rows * 4)
    datas = [torch.randint(0, 16, (rows, G), dtype=torch.uint8, device=dev) for _ in range(4)]
    t = timeit(lambda i: torch.ops.quanto.pack(datas[i % 4], 4))
    report("pack_int4", t, N * K + N * K // 2)
    packs = [torch.randint(0, 256, (rows // 2, G), dtype=torch.uint8, device=dev) for _ in range(6)]
    t = timeit(lambda i: torch.ops.quanto.unpack(packs[i % 6], 4))
    report("unpack_int4", t, N * K // 2 * 3)
    # fused freeze, 8 bit
    for name, dt in (("int8", torch.int8), ("e4m3", torch.float8_e4m3fn)):
        t = timeit(lambda i: torch.ops.quanto.quantize_qbytes_absmax(ws[i % nrot], dt))
        report(f"quantize_qbytes_absmax_bf16_{name}", t, N * K * 3 + N * 2)

    def ref_freeze8(i):
        w = ws[i % nrot]
        s = q.AbsmaxOptimizer()(w, qtype=q.qint8, axis=0)
        return torch.clamp(torch.round(w / s), -128, 127).to(torch.int8)

    t = timeit(ref_freeze8, iters=3, warmup=1, reps=3)
    report("reference_composition_aten_int8", t, N * K * 3 + N * 2)
    # activations: absmax + quantize_symmetric at [4096, 4096] bf16 (rotate 8 x 33 MB)
    xs = [torch.randn(4096, 4096, device=dev, dtype=torch.bfloat16) for _ in range(8)]
    t = timeit(lambda i: torch.ops.quanto.absmax(xs[i % 8]))
    report("absmax_bf16_4096x4096", t, 4096 * 4096 * 2)
    t = timeit(lambda i: torch.max(torch.abs(xs[i % 8])))
    report("reference_abs_max_aten", t, 4096 * 4096 * 2)
    sc = torch.tensor(0.03, device=dev, dtype=torch.bfloat16)
    for name, dt in (("int8", torch.int8), ("e4m3", torch.float8_e4m3fn)):
        t = timeit(lambda i: torch.ops.quanto.quantize_symmetric(xs[i % 8], dt, None, sc))
        report(f"quantize_symmetric_bf16_{name}_4096x4096", t, 4096 * 4096 * 3)
    srow = (torch.rand(4096, 1, device=dev) * 0.05 + 0.01).to(torch.bfloat16)
    t = timeit(lambda i: torch.ops.quanto.quantize_symmetric(xs[i % 8], torch.int8, 0, srow))
    report("quantize_symmetric_bf16_int8_axis0_4096x4096", t, 4096 * 4096 * 3)
    xh = [x.to(torch.float16) for x in xs]
    sh = sc.to(torch.float16)
    t = timeit(lambda i: torch.ops.quanto.quantize_symmetric(xh[i % 8], torch.int8, None, sh))
    report("quantize_symmetric_f16_int8_4096x4096", t, 4096 * 4096 * 3)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
