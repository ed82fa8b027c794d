"""Scoring kernels (kLCEScore epilogue in csrc/gemm_sm90.cu, lce_score_finalize in csrc/lce.cu) and
``LlamaForCausalLM.score`` on an H100.  Tolerances come from one measured run; the measured value is beside each."""
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import kernels as K
from opendiloco_b200.ops import tc_gemm as TC

pytestmark = pytest.mark.gpu

CSRC = Path(__file__).resolve().parent.parent / "opendiloco_b200" / "csrc"


def _run_kernels(x, w, labels):
    T, V = x.shape[0], w.shape[0]
    planes = TC.lce_planes(V)
    f32 = lambda n: torch.empty(n, dtype=torch.float32, device="cuda")  # noqa: E731
    pmax, psum, zlab = f32(planes * T), f32(planes * T), f32(T)
    pidx = torch.empty(planes * T, dtype=torch.int32, device="cuda")
    TC.lce_score(x, w, labels, pmax, psum, pidx, zlab)
    lp, lse = f32(T), f32(T)
    gr = torch.empty(T, dtype=torch.bool, device="cuda")
    am = torch.empty(T, dtype=torch.int32, device="cuda")
    K.lce_score_finalize(pmax, psum, pidx, zlab, planes, labels, lp, gr, lse, am)
    return lp, gr, lse, am


def _reference(x, w, labels):
    z = x.float() @ w.float().t()
    lse = torch.logsumexp(z, dim=-1)
    valid = labels >= 0
    zl = z.gather(1, labels.clamp(min=0)[:, None])[:, 0]
    return z, lse, torch.where(valid, zl - lse, torch.zeros_like(lse))


@pytest.mark.parametrize("h", [1024, 2048])
@pytest.mark.parametrize("V", [32000, 50264])
@pytest.mark.parametrize("T", [1, 127, 4000])
def test_score_kernels_match_fp32(T, V, h):
    g = torch.Generator(device="cuda").manual_seed(T * 7 + V + h)
    x = torch.randn(T, h, device="cuda", generator=g).bfloat16()
    w = (torch.randn(V, h, device="cuda", generator=g) * (3.0 / h ** 0.5)).bfloat16()     # logits of standard deviation ~3
    labels = torch.randint(0, V, (T,), device="cuda", generator=g)
    labels[::5] = -100
    lp, gr, lse, am = _run_kernels(x, w, labels)
    z, lse_ref, lp_ref = _reference(x, w, labels)
    e_lse = (lse - lse_ref).abs().max().item()
    e_lp = (lp - lp_ref).abs().max().item()
    top2 = z.topk(2, dim=-1).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-2
    print(f"T={T} V={V} h={h}: |lse err| {e_lse:.3g}, |logprob err| {e_lp:.3g}, clear-argmax rows {int(clear.sum())}/{T}")
    assert e_lse < 1e-3 and e_lp < 1e-3              # measured (H100, 12 shapes): lse <= 4.0e-5, logprob <= 5.3e-5
    assert torch.equal(am.long()[clear], z.argmax(dim=-1)[clear])
    valid = labels >= 0
    assert torch.equal(gr[clear], (valid & (am.long() == labels))[clear])
    assert torch.equal(lp[~valid], torch.zeros(int((~valid).sum()), device="cuda")) and not gr[~valid].any()


@pytest.mark.parametrize("V", [32000, 50264])
def test_score_kernel_exact_ties_take_the_lowest_index(V):
    T, h = 300, 1024
    g = torch.Generator(device="cuda").manual_seed(11)
    u = torch.randn(h, device="cuda", generator=g)
    x = (u + 0.3 * torch.randn(T, h, device="cuda", generator=g)).bfloat16()
    w = (0.02 * torch.randn(V, h, device="cuda", generator=g)).bfloat16()
    tied = [3, 700, V - 1]                               # three different 256-column planes, the last one partial for V = 50264
    w[tied] = (0.05 * u).bfloat16()                      # bit-identical rows: the row maximum, tied exactly
    labels = torch.tensor([3, 700, V - 1, 5], device="cuda").repeat(T // 4)
    lp, gr, lse, am = _run_kernels(x, w, labels)
    z, lse_ref, lp_ref = _reference(x, w, labels)
    assert bool((z[:, tied] == z.max(dim=-1, keepdim=True).values).all())
    assert torch.equal(am, torch.full_like(am, 3))
    assert torch.equal(gr, labels == 3)
    assert (lse - lse_ref).abs().max().item() < 1e-3


def test_score_kernel_exact_far_below_the_maximum():
    """Labels 150+ nats below the row maximum, where the training LCE clamps its exponent."""
    T, h, V = 256, 1024, 32000
    g = torch.Generator(device="cuda").manual_seed(12)
    u = torch.randn(h, device="cuda", generator=g)
    u = u / u.norm()
    x = (8 * u + 0.01 * torch.randn(T, h, device="cuda", generator=g)).bfloat16()
    w = (0.01 * torch.randn(V, h, device="cuda", generator=g)).bfloat16()
    w[17] = (16 * u).bfloat16()                          # z ~ +128
    w[20000] = (-12 * u).bfloat16()                      # z ~ -96: the label, ~220 nats below the maximum
    labels = torch.full((T,), 20000, device="cuda")
    labels[::7] = -100
    lp, gr, lse, am = _run_kernels(x, w, labels)
    z, lse_ref, lp_ref = _reference(x, w, labels)
    valid = labels >= 0
    gap = (z.max(dim=-1).values - z[:, 20000])[valid]
    assert gap.min().item() > 150
    assert torch.isfinite(lp).all() and torch.isfinite(lse).all()
    rel = ((lp - lp_ref).abs() / lp_ref.abs().clamp(min=1e-6))[valid].max().item()
    print(f"min gap {gap.min().item():.1f} nats, max relative logprob error {rel:.3g}")
    assert rel < 1e-3                                     # measured: 3.1e-6 at a 223-nat gap
    assert torch.equal(lp[~valid], torch.zeros(int((~valid).sum()), device="cuda")) and not gr.any()
    assert bool((am == 17).all())


def _layer_cfg(shape):
    if shape == "150m_layer":
        return LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=1, num_attention_heads=16, vocab_size=32000)
    return LlamaConfig(hidden_size=2048, intermediate_size=5632, num_hidden_layers=1, num_attention_heads=32, num_key_value_heads=4,
                       vocab_size=32000)


@pytest.mark.parametrize("shape", ["150m_layer", "1b_gqa_layer"])
def test_score_matches_fp32_engine(shape):
    cfg = _layer_cfg(shape)
    gpu = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=2)
    ref = LlamaForCausalLM(cfg, device="cuda", precision="32-true", seed=2)
    S = 300
    ids = torch.randint(0, cfg.vocab_size, (3, S), generator=torch.Generator().manual_seed(3)).cuda()
    mask = torch.ones_like(ids)
    mask[1, :77] = 0
    mask[2, 200:] = 0
    out = gpu.score(ids, attention_mask=mask)
    worst = 0.0
    for b in range(3):
        cols = mask[b].nonzero()[:, 0]
        lo, hi = int(cols[0]), int(cols[-1]) + 1
        with torch.no_grad():
            logits = ref(ids[b:b + 1, lo:hi]).logits[0].float()
        lp_ref = torch.log_softmax(logits, dim=-1)[:-1].gather(1, ids[b, lo + 1:hi, None])[:, 0]
        worst = max(worst, (out.logprobs[b, lo + 1:hi] - lp_ref).abs().max().item())
        assert out.logprobs[b, lo].item() == 0.0
    print(f"{shape}: max |logprob(bf16 kernels) - logprob(fp32 engine)| = {worst:.3g}")
    assert worst < 5e-2                  # measured: 0.018 (150m_layer), 0.029 (1b_gqa_layer): bf16 vs fp32 model


def test_padded_batch_equals_per_row_scoring():
    cfg = _layer_cfg("150m_layer")
    model = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=5)
    ids = torch.randint(0, cfg.vocab_size, (4, 333), generator=torch.Generator().manual_seed(6)).cuda()
    mask = torch.ones_like(ids)
    mask[0, :45] = 0
    mask[1, 131:] = 0
    mask[2, :7] = 0
    mask[2, 260:] = 0
    out = model.score(ids, attention_mask=mask)
    identical = True
    for b in range(4):
        cols = mask[b].nonzero()[:, 0]
        lo, hi = int(cols[0]), int(cols[-1]) + 1
        alone = model.score(ids[b:b + 1, lo:hi])
        err = (out.logprobs[b, lo:hi] - alone.logprobs[0]).abs().max().item()
        identical &= torch.equal(out.logprobs[b, lo:hi], alone.logprobs[0])
        assert err < 1e-5, (b, err)                      # measured: 0 (bit-identical)
        assert torch.equal(out.greedy[b, lo:hi], alone.greedy[0])
        assert not out.logprobs[b][mask[b] == 0].any() and not out.greedy[b][mask[b] == 0].any()
    print("padded batch bit-identical to per-row scoring:", identical)


def _our_kernel_names() -> set[str]:
    names = set()
    for src in CSRC.glob("*.cu"):
        names |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(", src.read_text()))
    return names


def test_score_launches_only_our_kernels():
    _in_fresh_process("_score_launches_only_our_kernels")


def _score_launches_only_our_kernels():
    cfg = _layer_cfg("1b_gqa_layer")
    model = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=0)
    ids = torch.randint(0, cfg.vocab_size, (3, 200), device="cuda")
    mask = torch.ones_like(ids)
    mask[0, :50] = 0
    model.score(ids, attention_mask=mask)
    torch.cuda.synchronize()
    ours = _our_kernel_names()
    assert {"lce_score_finalize_kernel", "gemm_kernel"} <= ours
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        model.score(ids, attention_mask=mask)
        torch.cuda.synchronize()
    gpu_events = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    kernels = [n for n in gpu_events if not n.startswith(("Memcpy", "Memset"))]   # copies of the inputs / outputs
    assert any("lce_score_finalize_kernel" in n for n in kernels), kernels
    foreign = [n for n in kernels if not any(re.search(rf"\b{k}\b", n) for k in ours)]
    assert not foreign, foreign


def test_score_does_not_disturb_training_graph():
    cfg = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4, vocab_size=512)
    model = LlamaForCausalLM(cfg, device="cuda", seed=0)
    batches = [torch.randint(3, 512, (4, 128), generator=torch.Generator().manual_seed(i)).cuda() for i in range(6)]
    for x in batches[:4]:
        model.forward_backward(x, x, 1.0)
    key = (4, 128, 1.0, True)
    g_obj = model.engine._graphs[key]["graph"]
    assert g_obj is not None
    ws_before = dict(model.engine._ws)
    state_before = [t.clone() for t in (model.arena.master, model.arena.grad, model.arena.shadow)]
    for B, S in ((2, 50), (3, 300), (5, 77)):                 # three new shapes: a workspace cache would evict
        model.score(batches[0][:B].repeat(1, 3)[:, :S])
    torch.cuda.synchronize()
    assert model.engine._graphs[key]["graph"] is g_obj
    assert model.engine._ws == ws_before
    for before, now in zip(state_before, (model.arena.master, model.arena.grad, model.arena.shadow)):
        assert torch.equal(before, now)
    for x in batches[4:]:
        loss = model.forward_backward(x, x, 1.0)
    assert model.engine._graphs[key]["graph"] is g_obj
    assert torch.isfinite(loss).all()


def _in_fresh_process(fn: str) -> None:
    """Run ``fn`` of this module in a new Python process and fail with its traceback if it fails.  Used by the tests that
    read kernel names from the CUDA profiler: late in a long pytest process the profiler intermittently records no GPU
    activity at all, while a fresh process records every launch."""
    here = Path(__file__).resolve()
    code = f"import sys; sys.path[:0] = [{str(here.parents[1])!r}, {str(here.parent)!r}]; import {here.stem}; {here.stem}.{fn}()"
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=here.parents[1], timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-6000:]
