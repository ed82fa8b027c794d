"""Rasterisation sweep of the GEMM at the Llama-150M micro-batch shapes (run once per ODB_GEMM_GROUP_M value; the
kernel reads the variable at its first launch).  L2 is flushed between timed launches."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from opendiloco_b200.ops import tc_gemm as T  # noqa: E402

BF = torch.bfloat16
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def timeit(fn, n=9):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(n):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return sorted(ts)[len(ts) // 2]


M = 32768
tag = f"group_m={os.environ.get('ODB_GEMM_GROUP_M', 'default16')} dx_group_m={os.environ.get('ODB_LCE_DX_GROUP_M', 'default16')}"
tot = 0.0
for name, N, K, nn in [("qkv fwd", 3072, 1024, False), ("o_proj fwd", 1024, 1024, False), ("gate-up fwd (plain)", 5376, 1024, False),
                       ("down fwd", 1024, 2688, False), ("o_proj dgrad", 1024, 1024, True), ("qkv dgrad", 1024, 3072, True),
                       ("gate-up dgrad", 1024, 5376, True)]:
    x = torch.randn(M, K, device="cuda").to(BF)
    w = (torch.randn(K, N, device="cuda") * 0.05).to(BF) if nn else (torch.randn(N, K, device="cuda") * 0.05).to(BF)
    out = torch.empty(M, N, device="cuda", dtype=BF)
    us = timeit((lambda: T.linear_nn(x, w, out)) if nn else (lambda: T.linear(x, w, out)))
    tot += us
    print(f"{tag:44s} {name:20s} {us:8.1f} us {2.0 * M * N * K / us / 1e6:7.0f} TF/s")
# LM-head dX on exponentials: K = vocabulary
V, h = 32000, 1024
e = torch.randn(M, V, device="cuda").to(BF)
w = (torch.randn(V, h, device="cuda") * 0.02).to(BF)
rs = torch.ones(M, device="cuda")
lab = torch.randint(0, V, (M,), device="cuda")
g = torch.ones(1, device="cuda")
dx = torch.empty(M, h, device="cuda", dtype=BF)
us = timeit(lambda: T.lce_dx(e, w, rs, lab, g, dx), n=5)
print(f"{tag:44s} {'LCE dX (K=32000)':20s} {us:8.1f} us {2.0 * M * V * h / us / 1e6:7.0f} TF/s")
print(f"{tag:44s} layer GEMM sum {tot:8.1f} us")
