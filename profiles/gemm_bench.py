"""wgmma GEMM family vs cuBLAS (torch.mm): numerics + CUDA-event timing at the Llama-150M / 1B shapes."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from opendiloco_b200.ops import tc_gemm as T, kernels as K
dev = "cuda"; BF = torch.bfloat16
torch.manual_seed(0)

def timeit(fn, n=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

def rel(a, b): return ((a.float() - b.float()).norm() / b.float().norm()).item()

print("== plain TN GEMM")
for (M, N, Kd) in [(300, 520, 200), (128, 256, 64), (4096, 1024, 1024), (32768, 1024, 1024), (32768, 3072, 1024), (32768, 5376, 1024),
                   (32768, 1024, 2688), (2048, 32000, 1024), (16384, 2560, 2048), (16384, 2048, 5632)]:
    x = torch.randn(M, Kd, device=dev).to(BF); w = (torch.randn(N, Kd, device=dev) * 0.05).to(BF)
    ref = torch.mm(x, w.t())
    out = T.linear(x, w)
    torch.cuda.synchronize()
    err = rel(out, ref)
    t1 = timeit(lambda: T.linear(x, w, out)); t0 = timeit(lambda: torch.mm(x, w.t(), out=ref))
    fl = 2 * M * N * Kd
    print(f"M{M} N{N} K{Kd}: rel_err {err:.2e}  ours {t1*1e3:.1f}us {fl/t1/1e9:.0f} TF/s | cublas {t0*1e3:.1f}us {fl/t0/1e9:.0f} TF/s | ratio {t0/t1:.2f}")

print("== gate|up + SwiGLU epilogue")
for (M, I, Kd) in [(256, 128, 64), (32768, 2688, 1024), (16384, 5632, 2048)]:
    x = torch.randn(M, Kd, device=dev).to(BF); w = (torch.randn(2 * I, Kd, device=dev) * 0.05).to(BF)
    gu_ref = torch.mm(x, w.t()); act_ref = K.swiglu_fwd(gu_ref)
    gu = torch.empty_like(gu_ref); act = torch.empty_like(act_ref)
    T.linear_swiglu(x, w, gu, act); torch.cuda.synchronize()
    t1 = timeit(lambda: T.linear_swiglu(x, w, gu, act))
    t0 = timeit(lambda: (torch.mm(x, w.t(), out=gu_ref), K.swiglu_fwd(gu_ref, out=act_ref)))
    print(f"M{M} I{I} K{Kd}: gu err {rel(gu, gu_ref):.2e} act err {rel(act, act_ref):.2e}  fused {t1*1e3:.1f}us | cublas+kernel {t0*1e3:.1f}us | ratio {t0/t1:.2f}")

print("== qkv + RoPE epilogue")
for (B, S, Hq, Hkv, Kd) in [(2, 128, 4, 4, 256), (32, 1024, 16, 16, 1024), (16, 1024, 32, 4, 2048)]:
    M = B * S; N = (Hq + 2 * Hkv) * 64
    x = torch.randn(M, Kd, device=dev).to(BF); w = (torch.randn(N, Kd, device=dev) * 0.05).to(BF)
    cos, sin = K.rope_tables(S, 64, 10000.0, dev)
    ref = torch.mm(x, w.t()); K.rope_(ref, cos, sin, S, Hq + Hkv, 64)
    out = torch.empty_like(ref)
    T.linear_qkv_rope(x, w, out, cos, sin, S, (Hq + Hkv) * 64); torch.cuda.synchronize()
    t1 = timeit(lambda: T.linear_qkv_rope(x, w, out, cos, sin, S, (Hq + Hkv) * 64))
    tmp = torch.empty_like(ref)
    t0 = timeit(lambda: (torch.mm(x, w.t(), out=tmp), K.rope_(tmp, cos, sin, S, Hq + Hkv, 64)))
    print(f"B{B} S{S} Hq{Hq} Hkv{Hkv} K{Kd}: err {rel(out, ref):.2e}  fused {t1*1e3:.1f}us | cublas+kernel {t0*1e3:.1f}us | ratio {t0/t1:.2f}")

print("== wgrad: dW(fp32) += dY^T X  (MN-major operands, split-K, TMA reduce-add)")
from opendiloco_b200.ops import gemm as G
for (Tn, N, Kd) in [(512, 256, 256), (1000, 520, 136), (32768, 1024, 1024), (32768, 3072, 1024), (32768, 5376, 1024), (32768, 1024, 2688),
                    (8192, 32000, 1024), (16384, 2560, 2048)]:
    dy = torch.randn(Tn, N, device=dev).to(BF); x = torch.randn(Tn, Kd, device=dev).to(BF)
    acc0 = torch.randn(N, Kd, device=dev)
    ref = acc0 + dy.float().t() @ x.float()
    out = acc0.clone(); T.wgrad_acc(dy, x, out); torch.cuda.synchronize()
    err = rel(out, ref)
    scratch = acc0.clone()
    t1 = timeit(lambda: T.wgrad_acc(dy, x, scratch)); t0 = timeit(lambda: torch.addmm(scratch, dy.t(), x, out_dtype=torch.float32, out=scratch))     # cuBLASLt, fp32 out, beta=1
    fl = 2 * Tn * N * Kd
    print(f"T{Tn} N{N} K{Kd}: rel_err {err:.2e}  ours {t1*1e3:.1f}us {fl/t1/1e9:.0f} TF/s | cublas {t0*1e3:.1f}us {fl/t0/1e9:.0f} TF/s | ratio {t0/t1:.2f}")
# three-source A (dq|dk|dv)
Tn, Kd = 32768, 1024
dq, dk, dv = (torch.randn(Tn, 1024, device=dev).to(BF) for _ in range(3)); x = torch.randn(Tn, Kd, device=dev).to(BF)
ref = torch.cat([dq, dk, dv], 1).float().t() @ x.float()
out = torch.zeros(3072, Kd, device=dev); T.wgrad_acc((dq, dk, dv), x, out); torch.cuda.synchronize()
print("3-source wgrad rel_err", rel(out, ref), "time", timeit(lambda: T.wgrad_acc((dq, dk, dv), x, out)) * 1e3, "us")

print("== down-proj dgrad + SwiGLU backward epilogue (d(act) never leaves the registers)")
for (M, I, Kd) in [(32768, 2688, 1024), (16384, 5632, 2048)]:
    dy = torch.randn(M, Kd, device=dev).to(BF); wt = (torch.randn(I, Kd, device=dev) * 0.05).to(BF)
    gu = torch.randn(M, 2 * I, device=dev).to(BF)
    dact = torch.empty(M, I, device=dev, dtype=BF)
    ref = K.swiglu_bwd(T.linear(dy, wt, dact), gu)
    fused = gu.clone(); T.linear_swiglu_bwd_t(dy, wt, fused); torch.cuda.synchronize()
    work = gu.clone()
    t1 = timeit(lambda: T.linear_swiglu_bwd_t(dy, wt, work))
    t0 = timeit(lambda: (torch.mm(dy, wt.t(), out=dact), K.swiglu_bwd(dact, work, work)))
    t2 = timeit(lambda: (T.linear(dy, wt, dact), K.swiglu_bwd(dact, work, work)))
    print(f"M{M} I{I} K{Kd}: err vs unfused {rel(fused, ref):.2e}  fused {t1*1e3:.1f}us | cublas+kernel {t0*1e3:.1f}us | own gemm+kernel {t2*1e3:.1f}us | ratio {t0/t1:.2f}")
