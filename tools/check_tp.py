"""Multi-rank check (torchrun, NCCL): column-parallel QLinear == single-GPU QLinear, BIT FOR BIT, for
* sharded canonical int4 weights + NCCL all-gather (`gather_columns`),
* the all-gather and rank synchronisation fused into the kernel (`FusedGather`: ring gemv M <= 8, wgmma kernel
  8 < M <= 128 -- tolerance there, its split of K depends on the shard shape --, persistent GEMM M > 128),
* a CHAIN of fused linears that synchronise only through the in-kernel flags (wait_input / no wait_output), eager and
  replayed from a CUDA graph.
Prints "TP CHECK OK" on rank 0 when every rank agrees.  Used by tests/test_gpu_qlinear.py (2 GPUs) and tools/gpu_*.sh."""
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "optimum-quanto_b200"))
import quanto_b200 as q  # noqa: E402
from bench import make_int4  # noqa: E402
from quanto_b200.parallel import ColumnParallelQLinear, FusedGather, shard_weight  # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
torch.manual_seed(0)
ok = True


def agree(flag):
    t = torch.tensor([1 if flag else 0], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    return bool(int(t.item()))


def close(a, b):
    d = (a.float() - b.float()).abs()
    return bool(torch.isfinite(a.float()).all()) and float(d.max()) <= 2.0 ** -6 * float(b.float().abs().max())


for (M, N, K) in ((8, 2048, 1024), (1, 14336, 4096), (40, 4096, 4096), (300, 4096, 2048), (1024, 14336, 4096)):
    lin = torch.nn.Linear(K, N, bias=True).to(torch.bfloat16)
    ql = q.QLinear.from_module(lin, weights=q.qint4)
    ql.freeze()
    x = torch.randn(M, K).to(torch.bfloat16).to(dev)
    y_full = ql.to(dev)(x)
    exact = not (8 < M <= 128)
    same_fn = torch.equal if exact else close
    tp = ColumnParallelQLinear(ql.weight, ql.bias.detach(), rank, world).to(dev)
    y_tp = tp(x)
    torch.cuda.synchronize()
    good = same_fn(y_tp, y_full)
    tpf = ColumnParallelQLinear(ql.weight, ql.bias.detach(), rank, world, fused=True).to(dev)
    for rep in range(3):  # the two symmetric buffers alternate
        y_f = tpf(x).clone()
        torch.cuda.synchronize()
        good = good and same_fn(y_f, y_full)
    good = agree(good)
    if rank == 0:
        print(f"M={M} N={N} K={K} world={world}: nccl + fused {'bit-identical' if exact else 'within tolerance'} "
              f"to the single-GPU linear: {good}", flush=True)
    ok = ok and good

# ---- a chain of fused linears, synchronised by the in-kernel flags only -------------------------------------------
for M in (1, 8, 32, 512):
    H, F = 4096, 14336
    # the graph and the buffers of the previous round must be gone BEFORE the next capture starts: a symmetric-memory
    # buffer whose last reference dies inside a capture is freed there, which CUDA forbids
    graph = yg = y = g1 = g2 = g3 = None
    import gc
    gc.collect()
    torch.cuda.synchronize()
    dist.barrier()
    w1, w2, w3 = make_int4(F, H, dev, 11), make_int4(H, F, dev, 12), make_int4(H, H, dev, 13)
    s1, s2, s3 = (shard_weight(w, rank, world) for w in (w1, w2, w3))
    x = (torch.randn(M, H, device=dev, generator=torch.Generator(device=dev).manual_seed(5)) * 0.1).to(torch.bfloat16)
    lin = torch.nn.functional.linear
    ref = lin(lin(lin(x, w1), w2), w3)  # single GPU
    g1, g2, g3 = FusedGather(F // world), FusedGather(H // world), FusedGather(H // world)

    def chain(xin):
        a = g1.forward(xin, s1, None, wait_input=True, wait_output=False)
        b = g2.forward(a, s2, None, wait_input=True, wait_output=False)
        return g3.forward(b, s3, None, wait_input=True, wait_output=True)

    # bit-identity needs kernels whose k-order does not depend on the shard shape: the ring gemv (whole-K ownership,
    # several passes over K when the activations do not fit shared memory; M <= 8) and the large-M GEMMs; the stream-K
    # wgmma kernel in between is checked against a tolerance
    exact = M <= 8 or M > 128
    same_fn = torch.equal if exact else close
    good = True
    for rep in range(3):
        y = chain(x).clone()
        torch.cuda.synchronize()
        good = good and same_fn(y, ref)
    dist.barrier()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        yg = chain(x)
    for rep in range(4):
        graph.replay()
        torch.cuda.synchronize()
        good = good and same_fn(yg, ref)
    good = agree(good)
    if rank == 0:
        print(f"chain of 3 fused linears, M={M}: eager x3 + graph replay x4 match the single-GPU chain: {good}", flush=True)
    ok = ok and good

dist.barrier()
if rank == 0:
    print("TP CHECK OK" if ok else "TP CHECK FAILED", flush=True)
dist.destroy_process_group()
sys.exit(0 if ok else 1)
