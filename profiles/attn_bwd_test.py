"""Our attention backward vs the fp32 math reference and cuDNN: numerics and timing."""
import math, os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from opendiloco_b200.ops import attention as A
A._LIB = "cudnn"      # attention_fwd / attention_bwd below = the cuDNN baseline; the tc_* entry points are ours
dev = "cuda"
def timeit(fn, n=10):
    for _ in range(2): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n
def rel(a, b): return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()
for (B, S, Hq, Hkv) in [(1, 128, 1, 1), (1, 256, 1, 1), (2, 256, 4, 2), (2, 1024, 4, 4), (32, 1024, 16, 16), (16, 1024, 32, 4)]:
    torch.manual_seed(0)
    qkv = torch.randn(B * S, (Hq + 2 * Hkv) * 64, device=dev).to(torch.bfloat16)
    out, lse = A.tc_attention_fwd(qkv, B, S, Hq, Hkv)
    dout = torch.randn_like(out)
    dq, dk, dv = A.tc_attention_bwd(dout, qkv, out, lse, B, S, Hq, Hkv)
    torch.cuda.synchronize()
    msg = f"B{B} S{S} Hq{Hq} Hkv{Hkv}:"
    if B * S <= 4096:
        qf = qkv.float()
        of, aux = A.attention_fwd(qf, B, S, Hq, Hkv, 64)
        dref = torch.empty_like(qf)
        A.attention_bwd(dout.float(), qf, of, aux, dref, B, S, Hq, Hkv, 64)
        rq, rk, rv = dref[:, :Hq * 64], dref[:, Hq * 64:(Hq + Hkv) * 64], dref[:, (Hq + Hkv) * 64:]
        msg += f" dq {rel(dq, rq):.2e} dk {rel(dk, rk):.2e} dv {rel(dv, rv):.2e}"
    else:
        o2, aux = A.attention_fwd(qkv, B, S, Hq, Hkv, 64)
        res = A.attention_bwd(dout, qkv, o2, aux, torch.empty_like(qkv), B, S, Hq, Hkv, 64, want_parts=True)
        msg += f" vs cudnn: dq {rel(dq, res[0]):.2e} dk {rel(dk, res[1]):.2e} dv {rel(dv, res[2]):.2e}"
        fl = 2.5 * 4 * S * S * Hq * 64 * B / 2
        packed = torch.empty_like(qkv)
        t1 = timeit(lambda: A.tc_attention_bwd(dout, qkv, out, lse, B, S, Hq, Hkv, dqkv=packed))   # pre-pass + main + post-pass
        t0 = timeit(lambda: A.attention_bwd(dout, qkv, o2, aux, torch.empty_like(qkv), B, S, Hq, Hkv, 64, want_parts=True))
        msg += f" | ours {t1*1e3:.0f}us {fl/t1/1e9:.0f} TF/s | cudnn {t0*1e3:.0f}us {fl/t0/1e9:.0f} TF/s"
    print(msg, flush=True)
