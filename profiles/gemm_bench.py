"""wgmma GEMM family vs cuBLAS (torch.mm): numerics + CUDA-event timing at the Llama-150M / 1B shapes.

    python profiles/gemm_bench.py [--root DIR] [--step-only]

--root DIR imports opendiloco_b200 from another built tree (e.g. an older commit, to compare two versions in one run);
--step-only times every GEMM of a Llama-150M micro-step (T = 32768: forwards, dgrads, the four layer weight gradients, the
LM-head forward, dX and dW) and prints one line per shape."""
import argparse, os, sys, torch
_ap = argparse.ArgumentParser()
_ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
_ap.add_argument("--step-only", action="store_true")
ARGS = _ap.parse_args()
sys.path.insert(0, os.path.abspath(ARGS.root))
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


def step_shapes(Tn=32768, h=1024, I=2688, V=32000, S=1024):
    """Every GEMM of a Llama-150M micro-step at Tn tokens: microseconds (median of 5 timings of 20 calls) and TFLOP/s."""
    x = torch.randn(Tn, h, device=dev).to(BF)
    rows = []
    def run(name, fn, flops):
        fn(); torch.cuda.synchronize()
        ts = sorted(timeit(fn) for _ in range(5))
        rows.append((name, ts[2] * 1e3, flops / (ts[2] * 1e-3) / 1e12, (ts[-1] - ts[0]) * 1e3))
    w_qkv = (torch.randn(3 * h, h, device=dev) * 0.05).to(BF); qkv = torch.empty(Tn, 3 * h, device=dev, dtype=BF)
    cos, sin = K.rope_tables(S, 64, 10000.0, dev)
    run("qkv_rope fwd K1024", lambda: T.linear_qkv_rope(x, w_qkv, qkv, cos, sin, S, 2 * h), 2 * Tn * 3 * h * h)
    w_o = (torch.randn(h, h, device=dev) * 0.05).to(BF); o = torch.empty(Tn, h, device=dev, dtype=BF)
    run("o fwd K1024", lambda: T.linear(x, w_o, o), 2 * Tn * h * h)
    w_gu = (torch.randn(2 * I, h, device=dev) * 0.05).to(BF)
    gu = torch.empty(Tn, 2 * I, device=dev, dtype=BF); act = torch.empty(Tn, I, device=dev, dtype=BF)
    run("gate|up swiglu fwd K1024", lambda: T.linear_swiglu(x, w_gu, gu, act), 2 * Tn * 2 * I * h)
    w_d = (torch.randn(h, I, device=dev) * 0.05).to(BF)
    run("down fwd K2688", lambda: T.linear(act, w_d, o), 2 * Tn * h * I)
    dy = torch.randn(Tn, h, device=dev).to(BF); gu0 = torch.randn(Tn, 2 * I, device=dev).to(BF)
    run("down dgrad+swiglu bwd K1024", lambda: T.linear_swiglu_bwd(dy, w_d, gu0), 2 * Tn * I * h)
    run("gate|up dgrad (nn) K5376", lambda: T.linear_nn(gu0, w_gu, o), 2 * Tn * h * 2 * I)
    run("o dgrad (nn) K1024", lambda: T.linear_nn(dy, w_o, o), 2 * Tn * h * h)
    dqkv = torch.randn(Tn, 3 * h, device=dev).to(BF)
    run("qkv dgrad (nn) K3072", lambda: T.linear_nn(dqkv, w_qkv, o), 2 * Tn * h * 3 * h)
    for (n, k, a) in [(3 * h, h, dqkv), (h, h, dy), (2 * I, h, gu0), (h, I, dy)]:
        b = x if k == h else act
        dw = torch.zeros(n, k, device=dev)
        run(f"wgrad N{n} K{k}", lambda a=a, b=b, dw=dw: T.wgrad_acc(a, b, dw), 2 * Tn * n * k)
    w_lm = (torch.randn(V, h, device=dev) * 0.02).to(BF)
    shift = torch.zeros(Tn, device=dev)
    planes = (V + 255) // 256
    partials = torch.empty(planes * Tn, device=dev); e = torch.empty(Tn, V, device=dev, dtype=BF)
    run("lce_fwd store=1 K1024", lambda: T.lce_fwd(x, w_lm, shift, partials, e), 2 * Tn * V * h)
    rs = torch.full((Tn,), 1e-3, device=dev); lab = torch.randint(0, V, (Tn,), device=dev); gs = torch.ones((), device=dev)
    run("lce_dx K32000", lambda: T.lce_dx(e, w_lm, rs, lab, gs, o), 2 * Tn * V * h)
    dw_lm = torch.zeros(V, h, device=dev)
    run(f"lce dW wgrad N{V} K{h}", lambda: T.wgrad_acc(e, x, dw_lm), 2 * Tn * V * h)
    for name, us, tf, spread in rows:
        print(f"STEP {name:32s} {us:9.1f} us {tf:6.1f} TF/s  (spread {spread:.1f} us)")


if ARGS.step_only:
    step_shapes()
    sys.exit(0)

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
