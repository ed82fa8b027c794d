"""precision="fp8-mixed" on the H100: the amax / cast kernels against the references bit for bit, every FP8 GEMM export
against the project's bf16 kernel on the quantised-dequantised (QDQ) operands, the fp32 promotion of long reductions, the
engine against 32-true / bf16-mixed, graph replay, the kernels a micro-step launches, and a short convergence run."""
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import fp8 as F
from opendiloco_b200.ops import kernels as K
from opendiloco_b200.ops import tc_gemm as TC

pytestmark = pytest.mark.gpu
CSRC = Path(__file__).resolve().parent.parent / "opendiloco_b200" / "csrc"
WIDTHS = {"150m": dict(h=1024, I=2688, qkv=3072, q=1024, rot=32), "1b_gqa": dict(h=2048, I=5632, qkv=2560, q=2048, rot=36)}


def _rel(a: torch.Tensor, b: torch.Tensor) -> float:
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30)).item()


def _q(x: torch.Tensor, fmt):
    """Kernel-quantised copy (row-major) and its inv scale."""
    slot, inv = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    out = torch.empty(x.shape, dtype=fmt, device="cuda")
    F.quantize(x.contiguous(), slot, inv, fmt, out=out)
    return out, inv


def _data(rows, cols, seed, spread=True):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(rows, cols, device="cuda", generator=g)
    if spread:     # magnitudes over many binades, so that FP8 subnormals and every exponent are exercised
        x = x * torch.exp2(torch.randint(-12, 4, (rows, cols), device="cuda", generator=g).float())
    return x.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------ casts
@pytest.mark.parametrize("fmt", [F.E4M3, F.E5M2], ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("shape", [(2048, 1024), (2048, 2688), (3072, 1024), (2048, 2048), (1024, 5632), (2560, 2048)])
def test_cast_is_bit_exact(fmt, shape):
    x = _data(*shape, seed=shape[1])
    slot, inv = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    out = torch.empty(shape, dtype=fmt, device="cuda")
    out_t = torch.empty(shape[::-1], dtype=fmt, device="cuda")
    F.quantize(x, slot, inv, fmt, out=out, out_t=out_t)
    q, iv = F.quantize_ref(x.cpu(), fmt)
    assert slot.item() == x.float().abs().max().item()
    assert inv.item() == iv.item()
    assert torch.equal(out.view(torch.uint8).cpu(), q.view(torch.uint8))
    assert torch.equal(out_t.view(torch.uint8).cpu(), q.view(torch.uint8).t())
    # a second cast from the same slot (the backward's transposed weight copy) writes the same bytes
    out_t2 = torch.empty_like(out_t)
    F.cast(x, slot, fmt, inv, out_t=out_t2)
    assert torch.equal(out_t2.view(torch.uint8), out_t.view(torch.uint8))


@pytest.mark.parametrize("fmt", [F.E4M3, F.E5M2], ids=["e4m3", "e5m2"])
@pytest.mark.parametrize("bad", [float("inf"), float("-inf"), float("nan")])
def test_cast_of_non_finite_tensor_is_nan(fmt, bad):
    x = _data(256, 512, seed=5)
    x[17, 300] = bad
    slot, inv = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    out = torch.empty(x.shape, dtype=fmt, device="cuda")
    out_t = torch.empty(x.shape[::-1], dtype=fmt, device="cuda")
    F.quantize(x, slot, inv, fmt, out=out, out_t=out_t)
    assert not torch.isfinite(slot).any() and torch.isnan(inv).all()
    assert (out.view(torch.uint8) == 0x7F).all() and (out_t.view(torch.uint8) == 0x7F).all()


def test_amax_of_zeros_gives_scale_one_and_slot_is_reset():
    x = torch.zeros(128, 256, dtype=torch.bfloat16, device="cuda")
    slot = torch.full((1,), 123.0, device="cuda")
    inv = torch.zeros(1, device="cuda")
    out = torch.empty(x.shape, dtype=F.E4M3, device="cuda")
    F.quantize(x, slot, inv, F.E4M3, out=out)
    assert slot.item() == 0.0 and inv.item() == 1.0 and (out.view(torch.uint8) == 0).all()


# ------------------------------------------------------------------------------------------------ GEMMs
# Normwise relative error of each FP8 export against the bf16 kernel on the QDQ operands (same products, different
# accumulation order and bf16 output rounding).  Measured on an H100 80GB HBM3 (400 W) at both widths: 6.2e-4 to 7.9e-4
# for the bf16 outputs, 1.1e-3 for the SwiGLU activation; wgrad (fp32 output) 1.0e-4 - inside each 128-deep k-block the
# tensor core accumulates FP8 products with fewer mantissa bits than fp32.
GEMM_TOL, WGRAD_TOL = 5e-3, 5e-4


@pytest.mark.parametrize("width", list(WIDTHS))
def test_fp8_gemms_match_bf16_kernels_on_qdq_operands(width):
    w = WIDTHS[width]
    T, h, I, n_qkv = 2048, w["h"], w["I"], w["qkv"]
    S = 1024
    errs = {}
    # forward projection (tn, e4m3 A) and dgrad (tn, e5m2 A)
    for name, fmt_a, (M, N, Kd) in (("tn_fwd", F.E4M3, (T, h, w["q"])), ("tn_dgrad", F.E5M2, (T, h, 2 * I))):
        a, ia = _q(_data(M, Kd, 1, spread=False), fmt_a)
        b, ib = _q(_data(N, Kd, 2, spread=False) * 0.05, F.E4M3)
        out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
        F.linear(a, b, ia, ib, out)
        errs[name] = _rel(out, TC.linear(F.dequantize(a, ia), F.dequantize(b, ib)))
    # fused QKV + RoPE
    x, ix = _q(_data(T, h, 3, spread=False), F.E4M3)
    wq, iw = _q(_data(n_qkv, h, 4, spread=False) * 0.05, F.E4M3)
    cos, sin = K.rope_tables(S, 64, 10000.0, "cuda")
    got = torch.empty(T, n_qkv, dtype=torch.bfloat16, device="cuda")
    ref = torch.empty_like(got)
    F.linear_qkv_rope(x, wq, ix, iw, got, cos, sin, S, w["rot"], 64)
    TC.linear_qkv_rope(F.dequantize(x, ix), F.dequantize(wq, iw), ref, cos, sin, S, w["rot"] * 64)
    errs["qkv_rope"] = _rel(got, ref)
    # SwiGLU forward
    wg, ig = _q(_data(2 * I, h, 5, spread=False) * 0.05, F.E4M3)
    gu, act = torch.empty(T, 2 * I, dtype=torch.bfloat16, device="cuda"), torch.empty(T, I, dtype=torch.bfloat16, device="cuda")
    gu_r, act_r = torch.empty_like(gu), torch.empty_like(act)
    F.linear_swiglu(x, wg, ix, ig, gu, act)
    TC.linear_swiglu(F.dequantize(x, ix), F.dequantize(wg, ig), gu_r, act_r)
    errs["swiglu_gu"], errs["swiglu_act"] = _rel(gu, gu_r), _rel(act, act_r)
    # SwiGLU backward (dgrad of down with the transposed e4m3 weight)
    dy, idy = _q(_data(T, h, 6, spread=False), F.E5M2)
    wdt, iwd = _q(_data(I, h, 7, spread=False) * 0.05, F.E4M3)
    g1, g2 = gu_r.clone(), gu_r.clone()
    F.linear_swiglu_bwd(dy, wdt, idy, iwd, g1)
    TC.linear_swiglu_bwd_t(F.dequantize(dy, idy), F.dequantize(wdt, iwd), g2)
    errs["swiglu_bwd"] = _rel(g1, g2)
    # weight gradient on the transposed copies
    dyt, idt = _q(_data(h, T, 8, spread=False), F.E5M2)
    xt, ixt = _q(_data(I, T, 9, spread=False), F.E4M3)
    dw = torch.full((h, I), 0.25, device="cuda")
    dw_r = dw.clone()
    F.wgrad(dyt, xt, idt, ixt, dw)
    TC.wgrad_acc(F.dequantize(dyt, idt).t().contiguous(), F.dequantize(xt, ixt).t().contiguous(), dw_r)
    errs["wgrad"] = _rel(dw, dw_r)
    print(width, {k: f"{v:.2e}" for k, v in errs.items()})
    assert all(v < GEMM_TOL for k, v in errs.items() if k != "wgrad"), errs
    assert errs["wgrad"] < WGRAD_TOL, errs


# Long reduction: T = 32768 tokens in one weight-gradient GEMM against an fp64 product of the same FP8 values.  Measured on an
# H100 80GB HBM3 (400 W): 1.0e-4 with the fp32 promotion after every 128-deep k-block - the same as the 2048-token
# wgrad above, i.e. the in-tensor-core accumulation of one k-block, while the sum over k-blocks is fp32.  A build without
# the promotion was not measured.
def test_long_k_wgrad_promotes_to_fp32():
    T, N_out, K_out = 32768, 512, 512
    dyt, idt = _q(_data(N_out, T, 11, spread=False), F.E5M2)
    xt, ixt = _q(_data(K_out, T, 12, spread=False).abs(), F.E4M3)     # one-signed operand: errors add up instead of cancelling
    dw = torch.zeros(N_out, K_out, device="cuda")
    F.wgrad(dyt, xt, idt, ixt, dw)
    ref = F.dequantize(dyt, idt).double() @ F.dequantize(xt, ixt).double().t()
    err = _rel(dw, ref)
    print("long-K wgrad rel err", err)
    assert err < 5e-4


# ------------------------------------------------------------------------------------------------ engine
def _layer_cfg(shape):
    if shape == "150m_layer":
        return LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=1, num_attention_heads=16, vocab_size=32000)
    return LlamaConfig(hidden_size=2048, intermediate_size=5632, num_hidden_layers=1, num_attention_heads=32, num_key_value_heads=4,
                       vocab_size=32000)


# Measured on an H100 80GB HBM3 (400 W, ids below): loss within 4e-5 relative of 32-true at both widths; worst per-tensor
# gradient error (q_proj) 0.145 (150M) / 0.159 (1B-GQA) against 32-true and the same against bf16-mixed: the e5m2
# rounding of the gradients (2 mantissa bits) dominates.
@pytest.mark.parametrize("shape", ["150m_layer", "1b_gqa_layer"])
def test_fp8_layer_against_fp32_and_bf16(shape):
    cfg = _layer_cfg(shape)
    models = {p: LlamaForCausalLM(cfg, device="cuda", precision=p, seed=2) for p in ("32-true", "bf16-mixed", "fp8-mixed")}
    torch.manual_seed(3)
    ids = torch.randint(3, cfg.vocab_size, (4, 512), device="cuda")
    loss = {p: m.forward_backward(ids, ids, 1.0).item() for p, m in models.items()}
    ref, f8 = models["32-true"].arena, models["fp8-mixed"].arena
    bf = models["bf16-mixed"].arena
    e32 = {n: _rel(f8.g(n), ref.g(n)) for n in ref.slots}
    ebf = {n: _rel(f8.g(n), bf.g(n)) for n in ref.slots}
    w32, wbf = max(e32.items(), key=lambda kv: kv[1]), max(ebf.items(), key=lambda kv: kv[1])
    print(shape, loss, "worst vs fp32", w32, "worst vs bf16", wbf)
    assert abs(loss["fp8-mixed"] - loss["32-true"]) / loss["32-true"] < 5e-3
    assert w32[1] < 0.25 and wbf[1] < 0.25


def test_fp8_graph_replay_matches_eager():
    cfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=2, num_attention_heads=16, vocab_size=32000)
    g = LlamaForCausalLM(cfg, device="cuda", precision="fp8-mixed", seed=4)
    e = LlamaForCausalLM(cfg, device="cuda", precision="fp8-mixed", seed=4)
    torch.manual_seed(5)
    batches = [torch.randint(3, cfg.vocab_size, (4, 512), device="cuda") for _ in range(4)]
    for ids in batches:                     # 2 eager warm-ups, capture, replay
        g.arena.grad.zero_()
        e.arena.grad.zero_()
        lg = g.engine.forward_backward_graphed(ids, ids, 1.0).item()
        le = e.engine.forward_backward(ids, ids, 1.0).item()
        assert abs(lg - le) <= 1e-3 * abs(le), (lg, le)
    assert any(st.get("graph") is not None for st in g.engine._graphs.values())
    err = _rel(g.arena.grad, e.arena.grad)
    print("graph vs eager grad rel err", err)
    # split-K weight gradients reduce with fp32 atomics (run-to-run order), and a last-bit change of a bf16 value can move
    # an FP8 rounding: measured 5e-9 on an H100 80GB HBM3
    assert err < 5e-3


FP8_GEMM = re.compile(r"gemm_kernel<\d+, false, false, [12]>")     # demangled name of an FP8 instantiation


def _our_kernel_names() -> set[str]:
    names = set()
    for src in CSRC.glob("*.cu"):
        names |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(", src.read_text()))
    return names


def _gpu_events(model, ids):
    from torch.profiler import ProfilerActivity, profile

    model.engine.forward_backward(ids, ids, 1.0)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        model.engine.forward_backward(ids, ids, 1.0)
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_fp8_micro_step_adds_only_our_kernels():
    _in_fresh_process("_fp8_micro_step_adds_only_our_kernels")


def _fp8_micro_step_adds_only_our_kernels():
    """Every GPU activity of an fp8-mixed micro-step is one of the project's kernels, a memset (the amax slot reset) or
    something the bf16-mixed micro-step launches too (its few PyTorch glue ops); the FP8 GEMMs and casts are ours."""
    cfg = _layer_cfg("1b_gqa_layer")
    ids = torch.randint(3, cfg.vocab_size, (2, 512), device="cuda")
    ours = _our_kernel_names()
    assert {"amax_kernel", "cast_kernel", "gemm_kernel"} <= ours
    ev8 = _gpu_events(LlamaForCausalLM(cfg, device="cuda", precision="fp8-mixed", seed=0), ids)
    ev16 = set(_gpu_events(LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=0), ids))
    is_ours = lambda n: any(re.search(rf"\b{k}\b", n) for k in ours)  # noqa: E731
    foreign = [n for n in ev8 if not is_ours(n) and "Memset" not in n and n not in ev16]
    assert not foreign, foreign
    assert any("amax_kernel" in n for n in ev8) and any("cast_kernel" in n for n in ev8)
    assert any(FP8_GEMM.search(n) for n in ev8), "no FP8 GEMM instantiation ran"
    assert not any(re.search(r"cutlass|cublas|gemm(?!_kernel)|sm90_xmma", n, re.I) for n in ev8 if not is_ours(n))


# ------------------------------------------------------------------------------------------------ convergence
def _bigram_stream(steps, B, S, V, seed):
    """A learnable stream: each token follows a fixed successor table with probability 0.85, else a uniform draw from
    512 ids (seeded, generated on the device)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    vocab = torch.randperm(V, device="cuda", generator=g)[:512]
    succ = torch.randint(0, 512, (512,), device="cuda", generator=g)
    out = []
    for _ in range(steps):
        idx = torch.empty(B, S, dtype=torch.long, device="cuda")
        idx[:, 0] = torch.randint(0, 512, (B,), device="cuda", generator=g)
        noise = torch.randint(0, 512, (B, S), device="cuda", generator=g)
        keep = torch.rand(B, S, device="cuda", generator=g) < 0.85
        for s in range(1, S):
            idx[:, s] = torch.where(keep[:, s], succ[idx[:, s - 1]], noise[:, s])
        out.append(vocab[idx])
    return out


def _train(precision, batches, cfg):
    m = LlamaForCausalLM(cfg, device="cuda", precision=precision, seed=0)
    opt = torch.optim.AdamW(m.parameters(), lr=1e-3, weight_decay=0.0, foreach=True)
    losses = []
    for ids in batches:
        opt.zero_grad(set_to_none=False)
        losses.append(m.forward_backward(ids, ids, 1.0).item())
        opt.step()
        m.sync_compute_weights()
    return losses


# Measured on an H100 80GB HBM3 (400 W), two runs: loss 10.60 at step 1; mean over the last 20 of 200 steps 1.4573 / 1.4572
# (bf16-mixed) vs 1.4576 / 1.4590 (fp8-mixed), 0.02 % / 0.12 % apart.
def test_fp8_training_converges_like_bf16():
    cfg = LlamaConfig.from_pretrained("60m")
    batches = _bigram_stream(200, 8, 256, cfg.vocab_size, seed=0)
    lb = _train("bf16-mixed", batches, cfg)
    l8 = _train("fp8-mixed", batches, cfg)
    tail_b, tail_8 = sum(lb[-20:]) / 20, sum(l8[-20:]) / 20
    print("first", lb[0], l8[0], "last-20 mean", tail_b, tail_8)
    assert tail_b < 0.5 * lb[0], "the stream was not learned"
    assert abs(tail_8 - tail_b) / tail_b < 0.02


def _in_fresh_process(fn: str) -> None:
    """Run ``fn`` of this module in a new Python process and fail with its traceback if it fails.  Used by the tests that
    read kernel names from the CUDA profiler: late in a long pytest process the profiler intermittently records no GPU
    activity at all, while a fresh process records every launch."""
    here = Path(__file__).resolve()
    code = f"import sys; sys.path[:0] = [{str(here.parents[1])!r}, {str(here.parent)!r}]; import {here.stem}; {here.stem}.{fn}()"
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=here.parents[1], timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-6000:]
