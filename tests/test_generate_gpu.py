"""Decode kernels (csrc/decode_sm90.cu) and KV-cached generation on an H100."""
import math
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.generation import decode_state, prefill, step
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import decode as DK
from opendiloco_b200.ops import kernels as K

pytestmark = pytest.mark.gpu

CSRC = Path(__file__).resolve().parent.parent / "opendiloco_b200" / "csrc"
LENGTHS = [1, 63, 64, 65, 127, 128, 129, 1000, 2048]


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


@pytest.mark.parametrize("Hq,Hkv", [(16, 16), (32, 4)])
def test_decode_attention_matches_fp32(Hq, Hkv):
    D, Smax, B = 64, 2048, len(LENGTHS)
    g = torch.Generator(device="cuda").manual_seed(0)
    q = torch.randn(B, (Hq + 2 * Hkv) * D, device="cuda", generator=g).bfloat16()
    kc = torch.randn(B, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
    vc = torch.randn(B, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
    pos = torch.tensor(LENGTHS, dtype=torch.int32, device="cuda") - 1
    nch = DK.attn_chunks(Smax)
    part_o = torch.empty(B, Hq, nch, D, device="cuda")
    part_ml = torch.empty(B, Hq, nch, 2, device="cuda")
    out = torch.empty(B, Hq * D, dtype=torch.bfloat16, device="cuda")
    DK.attention(q, kc, vc, pos, out, Hq, Hkv, D, part_o, part_ml)
    ref = torch.empty(B, Hq * D, dtype=torch.float32, device="cuda")
    DK.attention(q.float(), kc.float(), vc.float(), pos, ref, Hq, Hkv, D)      # fp32: the PyTorch reference
    for b, n in enumerate(LENGTHS):
        r = _rel(out[b], ref[b])
        assert r < 5e-3, (n, r)


def test_rope_append_matches_reference():
    Hq, Hkv, D, Smax = 8, 2, 64, 512
    positions = [0, 5, 127, 128, 300, 511]
    B = len(positions)
    g = torch.Generator(device="cuda").manual_seed(1)
    qkv = torch.randn(B, (Hq + 2 * Hkv) * D, device="cuda", generator=g).bfloat16()
    kc = torch.randn(B, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
    vc = torch.randn(B, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
    cos, sin = K.rope_tables(Smax, D, 10000.0, "cuda")
    pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
    q_ref, kc_ref, vc_ref = qkv.cpu(), kc.cpu(), vc.cpu()
    DK.rope_append(q_ref, cos.cpu(), sin.cpu(), pos.cpu(), kc_ref, vc_ref, Hq, Hkv, D)
    # the reference itself is K.rope_ at position p (rows laid out as sequences of length p+1)
    for b, p in enumerate(positions):
        seq = torch.zeros(p + 1, qkv.shape[1], dtype=torch.bfloat16)
        seq[p] = qkv[b].cpu()
        K.rope_(seq, cos[: p + 1].cpu(), sin[: p + 1].cpu(), p + 1, Hq + Hkv, D)
        assert torch.equal(seq[p, : Hq * D], q_ref[b, : Hq * D])
    before_k, before_v = kc.clone(), vc.clone()
    DK.rope_append(qkv, cos, sin, pos, kc, vc, Hq, Hkv, D)
    assert _rel(qkv[:, : Hq * D], q_ref[:, : Hq * D].cuda()) < 4e-3
    rows, p_c = torch.arange(B), pos.cpu().long()
    rows_g, p_g = rows.cuda(), pos.long()
    assert _rel(kc[rows_g, :, p_g], kc_ref[rows, :, p_c].cuda()) < 4e-3
    assert torch.equal(vc[rows_g, :, p_g], vc_ref[rows, :, p_c].cuda())
    touched = torch.zeros(B, Smax, dtype=torch.bool, device="cuda")
    touched[rows_g, p_g] = True
    keep = ~touched[:, None, :, None].expand_as(kc)
    assert torch.equal(kc[keep], before_k[keep]) and torch.equal(vc[keep], before_v[keep])


def _sample(logits, do_sample=True, temperature=1.0, top_k=0, top_p=1.0, seed=0):
    B = logits.shape[0]
    ictl, fctl = DK.make_controls(do_sample, temperature, top_k, top_p, seed, 0, [], "cuda")
    z = lambda: torch.zeros(B, dtype=torch.int32, device="cuda")  # noqa: E731
    out = torch.zeros(B, 1, dtype=torch.int64, device="cuda")
    ids = torch.zeros(B, dtype=torch.int64, device="cuda")
    DK.sample(logits, ictl, fctl, z(), z(), z(), out, ids)
    assert torch.equal(out[:, 0], ids)
    return ids


def test_sampler_greedy_topk_topp_and_seed():
    V = 32000
    g = torch.Generator(device="cuda").manual_seed(2)
    logits = (3 * torch.randn(64, V, device="cuda", generator=g)).bfloat16()
    # planted ties: the maximum appears at two (or three) indices
    logits[0, 17] = logits[0, 31000] = 40.0
    logits[1, 5] = logits[1, 6] = logits[1, 30000] = 41.0
    logits[2, :] = 1.0
    assert torch.equal(_sample(logits, do_sample=False), logits.argmax(dim=-1))
    assert torch.equal(_sample(logits, top_k=1, temperature=0.7), logits.argmax(dim=-1))

    x = logits.float()
    rep = 16                                             # every row drawn many times in one call
    big = logits.repeat(rep, 1)
    for kw in (dict(top_k=50), dict(top_p=0.9), dict(top_k=200, top_p=0.5, temperature=0.7), dict(top_p=0.3, temperature=2.0)):
        kept = torch.isfinite(DK.warp_logits(x, kw.get("temperature", 1.0), kw.get("top_k", 0), kw.get("top_p", 1.0)))
        # the kernel keeps every token tied with the smallest kept value (bf16 logits tie often); the sort in torch keeps
        # only some of them, in sort order
        floor = x.masked_fill(~kept, float("inf")).min(dim=-1, keepdim=True).values
        allowed = x >= floor
        tok = _sample(big, seed=11, **kw).view(rep, -1)
        for r in range(rep):
            ok = allowed.gather(1, tok[r][:, None])[:, 0]
            assert bool(ok.all()), (kw, torch.nonzero(~ok))
    a = _sample(big, seed=3, top_p=0.95)
    assert torch.equal(a, _sample(big, seed=3, top_p=0.95))
    assert not torch.equal(a, _sample(big, seed=4, top_p=0.95))


def test_sampler_temperature_chi_square():
    scipy_stats = pytest.importorskip("scipy.stats")
    V, rows, T = 64, 200_000, 0.7
    row = torch.randn(V, generator=torch.Generator().manual_seed(5)).bfloat16()
    logits = row.cuda()[None].repeat(rows, 1)
    tok = _sample(logits, temperature=T, seed=1234)
    counts = torch.bincount(tok, minlength=V).cpu().double()
    expected = torch.softmax(row.float().double() / T, dim=0) * rows
    stat, p = scipy_stats.chisquare(counts.numpy(), expected.numpy())
    print("chi-square", stat, "p", p)
    assert p > 1e-3


def _layer_cfg(shape):
    if shape == "150m_layer":
        return LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=1, num_attention_heads=16, vocab_size=32000)
    return LlamaConfig(hidden_size=2048, intermediate_size=5632, num_hidden_layers=1, num_attention_heads=32, num_key_value_heads=4,
                       vocab_size=32000)


@pytest.mark.parametrize("shape", ["150m_layer", "1b_gqa_layer"])
def test_teacher_forced_logits_match_fp32_engine(shape):
    cfg = _layer_cfg(shape)
    gpu = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=2)
    ref = LlamaForCausalLM(cfg, device="cuda", precision="32-true", seed=2)
    lens, n = [200, 77], 12
    B = len(lens)
    full = torch.randint(3, cfg.vocab_size, (B, max(lens) + n), generator=torch.Generator().manual_seed(3)).cuda()
    ref_logits = []
    with torch.no_grad():
        for b, L in enumerate(lens):
            ref_logits.append(ref(full[b:b + 1, : L + n]).logits[0, L - 1:])          # positions L-1 .. L+n-1
    st = decode_state(gpu, B, 512)
    assert st.kernels
    st.set_controls(False, 1.0, 0, 1.0, 0, 0, [])
    Sp = 256
    ids = torch.zeros(B, Sp, dtype=torch.int64, device="cuda")
    for b, L in enumerate(lens):
        ids[b, :L] = full[b, :L]
    prefill(gpu, st, ids, torch.tensor(lens, dtype=torch.int32, device="cuda"))
    for t in range(n):
        for b in range(B):
            r = _rel(st.logits[b], ref_logits[b][t])
            assert r < 2e-2, (shape, t, b, r)
        st.ids.copy_(torch.stack([full[b, L + t] for b, L in enumerate(lens)]))
        step(gpu, st, graph=(t % 2 == 0))                # eager and graph-replayed steps alike


@pytest.mark.parametrize("shape", ["150m_layer", "1b_gqa_layer"])
def test_greedy_generate_graph_equals_eager(shape, monkeypatch):
    cfg = _layer_cfg(shape)
    model = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=4)
    ids = torch.randint(3, cfg.vocab_size, (3, 150), generator=torch.Generator().manual_seed(5)).cuda()
    mask = torch.ones_like(ids)
    mask[1, :40] = 0
    mask[2, :149] = 0
    monkeypatch.setenv("ODB_CUDA_GRAPH", "1")
    graphed = model.generate(ids, attention_mask=mask, max_new_tokens=40, eos_token_id=[])
    assert model.engine.decode_state.graph is not None
    monkeypatch.setenv("ODB_CUDA_GRAPH", "0")
    eager = model.generate(ids, attention_mask=mask, max_new_tokens=40, eos_token_id=[])
    assert torch.equal(graphed, eager)
    sampled = [model.generate(ids, attention_mask=mask, max_new_tokens=40, do_sample=True, top_p=0.9, seed=7, eos_token_id=[])
               for _ in range(2)]
    assert torch.equal(sampled[0], sampled[1])


def _our_kernel_names() -> set[str]:
    names = set()
    for src in CSRC.glob("*.cu"):
        names |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(", src.read_text()))
    return names


def test_decode_step_launches_only_our_kernels():
    _in_fresh_process("_decode_step_launches_only_our_kernels")


def _decode_step_launches_only_our_kernels():
    cfg = _layer_cfg("1b_gqa_layer")
    model = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=0)
    st = decode_state(model, 4, 256)
    st.set_controls(True, 0.8, 40, 0.9, 0, 0, [])
    ids = torch.randint(3, cfg.vocab_size, (4, 128), device="cuda")
    prefill(model, st, ids, torch.full((4,), 128, dtype=torch.int32, device="cuda"))
    step(model, st, graph=False)
    torch.cuda.synchronize()
    ours = _our_kernel_names()
    assert {"decode_attn_kernel", "sample_kernel", "rope_append_kernel"} <= ours
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        step(model, st, graph=False)
        torch.cuda.synchronize()
    gpu_events = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert gpu_events, "the profiler recorded no GPU activity"
    foreign = [n for n in gpu_events if not any(re.search(rf"\b{k}\b", n) for k in ours)]
    assert not foreign, foreign


def test_generate_does_not_disturb_training_graph():
    """generate between graphed training steps: the training graph is not recaptured, the workspace is not evicted, no
    weight, gradient or compute-weight bit changes, and training continues like a twin that never generated.  The twins
    agree to rounding only: the loss and gradient reductions of the training step use fp32 atomics."""
    cfg = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4, vocab_size=512)
    a = LlamaForCausalLM(cfg, device="cuda", seed=0)
    b = LlamaForCausalLM(cfg, device="cuda", seed=0)
    batches = [torch.randint(3, 512, (4, 128), generator=torch.Generator().manual_seed(i)).cuda() for i in range(6)]
    la, lb = [], []
    for x in batches[:4]:
        la.append(a.forward_backward(x, x, 1.0).item())
        lb.append(b.forward_backward(x, x, 1.0).item())
    key = (4, 128, 1.0, True)
    g_obj = a.engine._graphs[key]["graph"]
    assert g_obj is not None
    ws_before = dict(a.engine._ws)
    state_before = [t.clone() for t in (a.arena.master, a.arena.grad, a.arena.shadow)]
    a.generate(batches[0][:2, :50], max_new_tokens=30, do_sample=True, seed=1)
    torch.cuda.synchronize()
    assert a.engine._graphs[key]["graph"] is g_obj
    assert a.engine._ws == ws_before
    for before, now in zip(state_before, (a.arena.master, a.arena.grad, a.arena.shadow)):
        assert torch.equal(before, now)
    for x in batches[4:]:
        la.append(a.forward_backward(x, x, 1.0).item())
        lb.append(b.forward_backward(x, x, 1.0).item())
    assert a.engine._graphs[key]["graph"] is g_obj
    for u, v in zip(la, lb):
        assert abs(u - v) <= 1e-5 * abs(v), (la, lb)
    assert _rel(a.arena.grad, b.arena.grad) < 1e-4
    assert not math.isnan(la[-1])


def _in_fresh_process(fn: str) -> None:
    """Run ``fn`` of this module in a new Python process and fail with its traceback if it fails.  Used by the tests that
    read kernel names from the CUDA profiler: late in a long pytest process the profiler intermittently records no GPU
    activity at all, while a fresh process records every launch."""
    here = Path(__file__).resolve()
    code = f"import sys; sys.path[:0] = [{str(here.parents[1])!r}, {str(here.parent)!r}]; import {here.stem}; {here.stem}.{fn}()"
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=here.parents[1], timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-6000:]
