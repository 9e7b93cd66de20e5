"""Developer probe: int4 GEMM time at the shard widths of 1/2/4/8-way column parallelism (M = 4096, K = 4096)."""
import os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from helpers import cabi_qbits_mm, native
from quick_bench import timeit
dev = "cuda"
lib = native().load()
M, K, G = 4096, 4096, 128
x = torch.randn(M, K, device=dev, dtype=torch.bfloat16)
for N in (14336, 7168, 3584, 1792):
    packed = torch.randint(0, 256, (N // 2, K), dtype=torch.uint8, device=dev)
    scale = (torch.rand(N * K // G, device=dev) * 0.01 + 0.002).to(torch.bfloat16)
    shift = (scale.float() * 8).to(torch.bfloat16)
    for name, rows in (("64-row tiles", 64), ("128-row tiles", 128)):
        with native().test_override(native().OVR_TILE_M, rows):
            t = timeit(lambda: cabi_qbits_mm(x, packed, scale, shift, None, N, K, G, use_workspace=False), iters=20)
        print(f"N={N:6d} {name:18s} {t*1e6:8.1f} us  {2*M*N*K/t/1e12:7.1f} TF/s", flush=True)
