"""Our attention forward vs cuDNN / fp32 math: numerics and timing."""
import math, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from opendiloco_b200.ops import attention as A
A._LIB = "cudnn"      # attention_fwd / attention_bwd below = the cuDNN baseline; the tc_* entry points are ours
dev = "cuda"
def timeit(fn, n=10):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n
for (B, S, Hq, Hkv) in [(1, 128, 1, 1), (2, 256, 4, 2), (2, 1024, 4, 4), (32, 1024, 16, 16), (16, 1024, 32, 4)]:
    torch.manual_seed(0)
    qkv = torch.randn(B * S, (Hq + 2 * Hkv) * 64, device=dev).to(torch.bfloat16)
    out, lse = A.tc_attention_fwd(qkv, B, S, Hq, Hkv)
    torch.cuda.synchronize()
    ref, (lse_ref, _) = A.attention_fwd(qkv.float(), B, S, Hq, Hkv, 64)       # fp32 math path
    err = ((out.float() - ref).norm() / ref.norm()).item()
    lerr = (lse - lse_ref).abs().max().item()
    msg = f"B{B} S{S} Hq{Hq} Hkv{Hkv}: rel_err {err:.3e} lse_err {lerr:.2e}"
    if B * S >= 2048:
        fl = 4 * S * S * Hq * 64 * B / 2
        t1 = timeit(lambda: A.tc_attention_fwd(qkv, B, S, Hq, Hkv))
        t0 = timeit(lambda: A.attention_fwd(qkv, B, S, Hq, Hkv, 64))
        msg += f" | ours {t1*1e3:.0f}us {fl/t1/1e9:.0f} TF/s | cudnn {t0*1e3:.0f}us {fl/t0/1e9:.0f} TF/s"
    print(msg, flush=True)
