"""Developer benchmark of the fused HQQ freeze (csrc/hqq.cu, quanto::quantize_qbits_hqq) against HqqOptimizer running as
the torch composition on the same GPU (the reference's algorithm, optimum/quanto/tensor/optimizers/hqq_optimizer.py:60-87,
followed by the package's quantize_affine and packing of the frozen weight).  CUDA events; the two take turns in one process.
The composition syncs the host once per iteration (float() of the mean error), so it is timed as a whole call.

    python tools/bench_hqq.py > hqq_bench.json
"""
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "optimum-quanto_b200"))
import quanto_b200 as q  # noqa: E402
from quanto_b200.library import quantize_affine_any  # noqa: E402
from quanto_b200.tensor.grouped import group  # noqa: E402
from quanto_b200.tensor.packed import pack_weights  # noqa: E402

G = 128
SHAPES = [(4096, 4096), (1024, 4096), (14336, 4096), (4096, 14336)]
# Llama-3-8B: per decoder layer q, k, v, o, gate, up, down (out_features, in_features); 32 layers = 224 linears
LLAMA_LAYER = [(4096, 4096), (1024, 4096), (1024, 4096), (4096, 4096), (14336, 4096), (14336, 4096), (4096, 14336)]


def fused(w, qt):
    return torch.ops.quanto.quantize_qbits_hqq(w, qt.bits, G, False, 0.7, 10.0, 1.01, 20)


def composition(w, qt):
    scale, shift = q.HqqOptimizer().optimize(group(w, 0, G), qt, 0)
    data = quantize_affine_any(w, qt.bits, 0, G, scale, shift)
    return pack_weights(data, qt.bits), scale, shift


def time_call(fn, reps):
    """Milliseconds per call: CUDA events around `reps` calls, after one untimed call."""
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    torch.manual_seed(0)
    props = torch.cuda.get_device_properties(0)
    res = {"gpu": props.name, "group_size": G, "dtype": "bf16", "shapes": [], "llama3_8b_freeze": {}}
    for N, K in SHAPES:
        w = (torch.randn(N, K, device="cuda") * 0.02).to(torch.bfloat16)
        for qt in (q.qint4, q.qint2):
            f, c = [], []
            for _ in range(3):  # turns: fused, composition, fused, ...
                f.append(time_call(lambda: fused(w, qt), 10))
                c.append(time_call(lambda: composition(w, qt), 2))
            _, _, _, errors = fused(w, qt)
            res["shapes"].append({
                "N": N, "K": K, "qtype": qt.name, "fused_ms": min(f), "composition_ms": min(c),
                "speedup": min(c) / min(f), "accepted": int(errors[-1].item()),
                # the fused op reads the weight twice and stores 21 candidate shifts of 2 bytes per group row
                "fused_bytes": N * K * 2 * 2 + N * K * qt.bits // 8 + (N * K // G) * (2 * 21 * 2 + 4),
            })
        del w
    # freeze() of the 224 linears of Llama-3-8B (bf16, qint4, group 128) with HqqOptimizer on the device: the fused path
    # over 224 distinct weights (15 GB); the composition over one decoder layer, times 32 (an extrapolation)
    layers = [[q.QLinear.from_module(torch.nn.Linear(k, n, bias=False, device="cuda", dtype=torch.bfloat16),
                                     weights=q.qint4, optimizer=q.HqqOptimizer()) for n, k in LLAMA_LAYER]
              for _ in range(32)]
    with torch.no_grad():
        for name, mods, freeze_one in (("fused_224_s", [m for layer in layers for m in layer], lambda m: m.qweight),
                                       ("composition_one_layer_s", layers[0],
                                        lambda m: composition(m.weight.detach(), q.qint4))):
            freeze_one(mods[0])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for m in mods:
                freeze_one(m)
            torch.cuda.synchronize()
            res["llama3_8b_freeze"][name] = time.perf_counter() - t0
    res["llama3_8b_freeze"]["composition_224_extrapolated_s"] = 32 * res["llama3_8b_freeze"]["composition_one_layer_s"]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
