"""Library attention candidates on the GPU at the flagship shape (B=32,S=1024,H=16,D=64): flash-attn 2.8 vs cuDNN SDPA."""
import math, sys, os, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
B, S, H, D = 32, 1024, 16, 64
dev = "cuda"
qkv = torch.randn(B * S, 3 * H * D, device=dev).to(torch.bfloat16)
from opendiloco_b200.ops import attention as A

def timeit(fn, n=10):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

fl_f = 4 * S * S * H * D * B / 2
out, aux = A.attention_fwd(qkv, B, S, H, H, D)
dout = torch.randn_like(out); dqkv = torch.empty_like(qkv)
t = timeit(lambda: A.attention_fwd(qkv, B, S, H, H, D)); print(f"flash fwd {t:.3f} ms {fl_f/t/1e9:.0f} TF/s")
t = timeit(lambda: A.attention_bwd(dout, qkv, out, aux, dqkv, B, S, H, H, D)); print(f"flash bwd {t:.3f} ms {2.5*fl_f/t/1e9:.0f} TF/s")
q, k, v = A.split_qkv(qkv, B, S, H, H, D)
qt, kt, vt = (x.transpose(1, 2) for x in (q, k, v))
try:
    f = torch.ops.aten._scaled_dot_product_cudnn_attention
    r = f(qt, kt, vt, None, True, 0.0, True, False, scale=1/math.sqrt(D))
    o2 = r[0]
    print("cudnn out strides", o2.stride(), "max diff vs flash", (o2.transpose(1,2).reshape(B*S, H*D).float()-out.float()).abs().max().item())
    t = timeit(lambda: f(qt, kt, vt, None, True, 0.0, True, False, scale=1/math.sqrt(D))); print(f"cudnn fwd {t:.3f} ms {fl_f/t/1e9:.0f} TF/s")
    fb = torch.ops.aten._scaled_dot_product_cudnn_attention_backward
    do = dout.view(B, S, H, D).transpose(1, 2)
    def bwd():
        return fb(do, qt, kt, vt, r[0], r[1], r[6], r[7], None, r[2], r[3], r[4], r[5], 0.0, True, scale=1/math.sqrt(D))
    g = bwd()
    print("cudnn dq strides", g[0].stride())
    t = timeit(bwd); print(f"cudnn bwd {t:.3f} ms {2.5*fl_f/t/1e9:.0f} TF/s")
    A.attention_bwd(dout, qkv, out, aux, dqkv, B, S, H, H, D)
    dq = A.split_qkv(dqkv, B, S, H, H, D)[0]
    print("dq diff", (g[0].transpose(1,2).float()-dq.float()).abs().max().item())
except Exception as e:
    import traceback; traceback.print_exc()
# GQA variant
try:
    Hkv = 4; Hq = 32
    qkv2 = torch.randn(16 * S, (Hq + 2 * Hkv) * D, device=dev).to(torch.bfloat16)
    q, k, v = A.split_qkv(qkv2, 16, S, Hq, Hkv, D)
    r = torch.ops.aten._scaled_dot_product_cudnn_attention(q.transpose(1,2), k.transpose(1,2), v.transpose(1,2), None, True, 0.0, True, False, scale=1/math.sqrt(D))
    o3, _ = A.attention_fwd(qkv2, 16, S, Hq, Hkv, D)
    print("cudnn gqa ok, diff", (r[0].transpose(1,2).reshape(16*S, Hq*D).float()-o3.float()).abs().max().item())
except Exception as e:
    print("cudnn gqa failed:", type(e).__name__, str(e)[:200])
