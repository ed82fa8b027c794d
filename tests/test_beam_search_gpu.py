"""Beam search on an H100: the selection kernels against ``beam_step_reference``, the chunk table against physically
reordered caches, and ``generate(num_beams=...)`` end to end."""
import math
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from opendiloco_b200.models import generation as G
from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.generation import beam_prefill, beam_select, beam_state, beam_step
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import decode as DK

pytestmark = pytest.mark.gpu

CSRC = Path(__file__).resolve().parent.parent / "opendiloco_b200" / "csrc"
V = 32000


def _select_inputs(B, nb, K, M, t, n_eos, seed):
    """Random selection state at step t (histories: random before t, pad from t on; prompt 1 already done)."""
    g = torch.Generator().manual_seed(seed)
    rows = B * nb
    logits = (3 * torch.randn(rows, V, generator=g)).bfloat16()
    top = logits.float().topk(4, dim=1).indices
    eos = top[:, :2].flatten().unique()[:n_eos].tolist()                       # EOS ids that really are candidates
    eos += [V - 1 - i for i in range(n_eos - len(eos))]
    run_score = -4 * torch.rand(rows, generator=g)
    fin_score = -3 * torch.rand(rows, generator=g)
    fin_flag = (torch.rand(rows, generator=g) < 0.5).int()
    fin_score = torch.where(fin_flag.bool(), fin_score, torch.full_like(fin_score, DK.NEG))
    hist = torch.randint(0, V, (2, rows, M), generator=g, dtype=torch.int64).int()
    hist[:, :, t:] = 0
    state = dict(run_score=run_score, fin_score=fin_score, fin_flag=fin_flag, run_seq=hist.clone(), fin_seq=hist.flip(1).contiguous(),
                 unsat=torch.ones(B, dtype=torch.int32), done=torch.zeros(B, dtype=torch.int32),
                 tstep=torch.full((B,), t, dtype=torch.int32), pos=torch.randint(100, 200, (B,), generator=g).int().repeat_interleave(nb),
                 ids_next=torch.zeros(rows, dtype=torch.int64), parent=torch.zeros(rows, dtype=torch.int32))
    state["done"][1] = 1
    state["unsat"][2] = 0
    return logits, eos, state


def _near_tie(logits, state, nb, K):
    """The reference's top K + 1 scores of a live prompt hold two from different beams within 1e-3."""
    B = logits.shape[0] // nb
    s = (torch.log_softmax(logits.float(), -1) + state["run_score"][:, None]).view(B, -1)
    vals, idx = s.topk(K + 1, dim=1)
    beams = idx // V
    gap = (vals[:, :-1] - vals[:, 1:]).abs()
    return bool(((gap < 1e-3) & (beams[:, :-1] != beams[:, 1:])).any())


@pytest.mark.parametrize("n_eos", [1, 8])
@pytest.mark.parametrize("early_stopping", [0, 1, 2])
@pytest.mark.parametrize("at_limit", [False, True])
@pytest.mark.parametrize("nb", [4, 8])
def test_select_kernels_match_reference(n_eos, early_stopping, at_limit, nb):
    B, M = 4, 40
    t = M - 1 if at_limit else M - 2
    K = DK.beams_to_keep(nb, n_eos)
    seed = 0
    while True:
        logits, eos, st = _select_inputs(B, nb, K, M, t, n_eos, seed)
        if not _near_tie(logits, st, nb, K):
            break
        seed += 1
    ictl, _ = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, eos, "cpu")
    ref = {k: v.clone() for k, v in st.items()}
    DK.beam_step_reference(logits, ictl, nb, K, 1.3, early_stopping, M, **ref)
    gpu = {k: v.cuda() for k, v in st.items()}
    rows, nsp = B * nb, DK.beam_splits(V)
    part_ml = torch.empty(rows, nsp, 2, device="cuda")
    cand_v = torch.empty(rows, nsp, K, device="cuda")
    cand_i = torch.empty(rows, nsp, K, dtype=torch.int32, device="cuda")
    DK.beam_select(logits.cuda(), ictl.cuda(), nb, K, 1.3, early_stopping, M, **gpu, part_ml=part_ml, cand_v=cand_v, cand_i=cand_i)
    torch.cuda.synchronize()
    for k in ("fin_flag", "run_seq", "fin_seq", "unsat", "done", "tstep", "pos", "ids_next", "parent"):
        assert torch.equal(gpu[k].cpu(), ref[k]), k
    for k in ("run_score", "fin_score"):
        assert torch.allclose(gpu[k].cpu(), ref[k], atol=1e-5, rtol=1e-6), (k, (gpu[k].cpu() - ref[k]).abs().max())
    assert torch.equal(gpu["pos"].cpu(), st["pos"] + (st["done"] == 0).int().repeat_interleave(nb))


@pytest.mark.parametrize("Hq,Hkv", [(16, 16), (32, 4)])
def test_table_attention_is_bit_identical_to_gathered_cache(Hq, Hkv):
    D, Smax, rows = 64, 1024, 8
    g = torch.Generator(device="cuda").manual_seed(0)
    q = torch.randn(rows, (Hq + 2 * Hkv) * D, device="cuda", generator=g).bfloat16()
    kc = torch.randn(rows, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
    vc = torch.randn(rows, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
    nch = DK.attn_chunks(Smax)
    table = torch.randint(0, rows, (rows, nch), device="cuda", generator=g, dtype=torch.int64).int()
    pos = torch.tensor([0, 127, 128, 129, 500, 640, 1000, 1023], dtype=torch.int32, device="cuda")
    part_o, part_ml = torch.empty(rows, Hq, nch, D, device="cuda"), torch.empty(rows, Hq, nch, 2, device="cuda")
    a = torch.empty(rows, Hq * D, dtype=torch.bfloat16, device="cuda")
    b = torch.empty_like(a)
    DK.attention(q, kc, vc, pos, a, Hq, Hkv, D, part_o, part_ml, table=table)
    DK.attention(q, DK.gather_chunks(kc, table), DK.gather_chunks(vc, table), pos, b, Hq, Hkv, D, part_o, part_ml)
    assert torch.equal(a, b)


@pytest.mark.parametrize("nb", [4, 8])
def test_reorder_through_table_equals_physical_reorder(nb):
    L, Hkv, D, Smax, B, steps = 2, 2, 64, 512, 2, 320
    rows = B * nb
    g = torch.Generator().manual_seed(nb)
    kv_t = torch.randn(L, 2, rows, Hkv, Smax, D, generator=g).bfloat16().cuda()
    kv_r = kv_t.clone()
    table = torch.arange(rows, dtype=torch.int32, device="cuda")[:, None].repeat(1, Smax // 128).contiguous()
    pos = torch.tensor([60, 150], dtype=torch.int32).repeat_interleave(nb).cuda()
    moved = 0
    for s in range(steps):
        # the decode step writes each row's new K/V at its position, into its own row
        new = torch.randn(L, 2, rows, Hkv, D, generator=g).bfloat16().cuda()
        idx = torch.arange(rows, device="cuda")
        kv_t[:, :, idx, :, pos.long()] = new.permute(2, 0, 1, 3, 4)
        kv_r[:, :, idx, :, pos.long()] = new.permute(2, 0, 1, 3, 4)
        pos += 1
        par = []
        for b in range(B):
            kind = (s + b) % 4
            if kind == 0:
                ch = torch.randint(0, nb, (nb,), generator=g)                       # copies
            elif kind == 1:
                ch = torch.randperm(nb, generator=g)                                # swaps and cycles
            elif kind == 2:
                ch = torch.roll(torch.arange(nb), 1)                                # one cycle over all beams
            else:
                ch = torch.arange(nb)                                               # every beam keeps itself
            par.append(ch + b * nb)
        parent = torch.cat(par).int().cuda()
        moved += int((parent != idx.int()).sum())
        DK.beam_reorder(kv_t, table, parent, pos, nb)
        DK.beam_reorder_reference(kv_r, parent)
        if s % 40 == 39 or s == steps - 1:
            torch.cuda.synchronize()
            for l in range(L):
                for kv in range(2):
                    seen = DK.gather_chunks(kv_t[l, kv], table)
                    for r in range(rows):
                        p = int(pos[r])
                        assert torch.equal(seen[r, :, :p], kv_r[l, kv, r, :, :p]), (s, l, kv, r)
    assert moved > 0 and int(pos.max()) > 3 * 128


def test_reorder_at_the_end_of_the_cache_stays_inside_the_table():
    """generate() ends at position P + max_new_tokens - 1 = Smax - 1 when P + max_new_tokens is a multiple of 128; even a
    full cache (position Smax) writes no table entry past the rows.  A sentinel row after the table must not change."""
    L, Hkv, D, Smax, B, nb = 2, 2, 64, 256, 2, 4
    rows, nch = B * nb, Smax // 128
    g = torch.Generator().manual_seed(3)
    kv_t = torch.randn(L, 2, rows, Hkv, Smax, D, generator=g).bfloat16().cuda()
    kv_r = kv_t.clone()
    full = torch.full((rows + 1, nch), -7, dtype=torch.int32, device="cuda")
    table = full[:rows]
    table.copy_(torch.arange(rows, dtype=torch.int32, device="cuda")[:, None].expand(rows, nch))
    pos = torch.tensor([Smax - 1, Smax], dtype=torch.int32).repeat_interleave(nb).cuda()
    for perm in ([1, 0, 3, 2], [2, 2, 0, 1], [3, 0, 1, 2]):                    # swaps, copies, a cycle
        parent = torch.cat([torch.tensor(perm) + b * nb for b in range(B)]).int().cuda()
        DK.beam_reorder(kv_t, table, parent, pos, nb)
        DK.beam_reorder_reference(kv_r, parent)
    torch.cuda.synchronize()
    assert bool((full[rows] == -7).all())
    for l in range(L):
        for kv in range(2):
            seen = DK.gather_chunks(kv_t[l, kv], table)
            for r in range(rows):
                p = int(pos[r])
                assert torch.equal(seen[r, :, :p], kv_r[l, kv, r, :, :p]), (l, kv, r)


def _layer_cfg(shape):
    if shape == "150m_layer":
        return LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=1, num_attention_heads=16, vocab_size=V)
    return LlamaConfig(hidden_size=2048, intermediate_size=5632, num_hidden_layers=1, num_attention_heads=32, num_key_value_heads=4,
                       vocab_size=V)


def _prompts(n=3, P=150, seed=5):
    ids = torch.randint(3, V, (n, P), generator=torch.Generator().manual_seed(seed)).cuda()
    mask = torch.ones_like(ids)
    mask[1, :40] = 0
    mask[2, :P - 1] = 0
    return ids, mask


@pytest.mark.parametrize("shape", ["150m_layer", "1b_gqa_layer"])
def test_graph_equals_eager(shape, monkeypatch):
    model = LlamaForCausalLM(_layer_cfg(shape), device="cuda", precision="bf16-mixed", seed=4)
    ids, mask = _prompts()
    kw = dict(attention_mask=mask, max_new_tokens=40, num_beams=4, num_return_sequences=4, eos_token_id=[17, 99, 1000],
              length_penalty=0.8, return_dict_in_generate=True)
    monkeypatch.setenv("ODB_CUDA_GRAPH", "1")
    graphed = model.generate(ids, **kw)
    assert model.engine.beam_state.kernels and model.engine.beam_state.graph is not None
    monkeypatch.setenv("ODB_CUDA_GRAPH", "0")
    eager = model.generate(ids, **kw)
    assert torch.equal(graphed.sequences, eager.sequences)
    assert torch.equal(graphed.sequences_scores, eager.sequences_scores)


@pytest.mark.parametrize("shape", ["150m_layer", "1b_gqa_layer"])
def test_kernels_equal_reference_program(shape, monkeypatch):
    """With o_proj zeroed, attention adds nothing to the residual stream, so both programs see the same logits and the
    selection, bookkeeping and output must agree exactly.  Beam search compares accumulated scores across beams, so with
    attention in play the two programs' bf16 rounding differences flip near-ties; the score() oracle below covers that."""
    model = LlamaForCausalLM(_layer_cfg(shape), device="cuda", precision="bf16-mixed", seed=6)
    with torch.no_grad():
        dict(model.named_parameters())["model.layers.0.self_attn.o_proj.weight"].zero_()
    model.arena.sync_shadow()
    ids, mask = _prompts()
    kw = dict(attention_mask=mask, max_new_tokens=40, num_beams=4, num_return_sequences=2, eos_token_id=[17, 99, 1000],
              length_penalty=1.5, early_stopping=True, return_dict_in_generate=True)
    got = model.generate(ids, **kw)
    assert model.engine.beam_state.kernels
    model.engine.beam_state = None
    with monkeypatch.context() as m:
        m.setattr(DK, "usable", lambda *a, **k: False)                   # the whole program on the PyTorch references
        ref = model.generate(ids, **kw)
        assert not model.engine.beam_state.kernels
    model.engine.beam_state = None
    assert torch.equal(got.sequences, ref.sequences)
    assert torch.allclose(got.sequences_scores, ref.sequences_scores, atol=1e-5, rtol=0)


@pytest.mark.parametrize("shape", ["150m_layer", "1b_gqa_layer"])
def test_chunk_table_program_equals_physical_reorder_program(shape, monkeypatch):
    """The full kernel program with attention in play, once through the chunk table and once with the table off and the
    caches reordered physically after every step: the same attention kernel reads the same keys, so the sequences and
    scores must be bit-identical.  P + max_new_tokens = 256 = Smax: the last step reorders at position Smax - 1."""
    model = LlamaForCausalLM(_layer_cfg(shape), device="cuda", precision="bf16-mixed", seed=8)
    ids, mask = _prompts(P=128)
    n_new = 128
    kw = dict(attention_mask=mask, max_new_tokens=n_new, num_beams=4, num_return_sequences=4, eos_token_id=[17, 99, 1000],
              length_penalty=1.2, early_stopping="never", return_dict_in_generate=True)
    monkeypatch.setenv("ODB_CUDA_GRAPH", "1")
    got = model.generate(ids, **kw)
    bs = model.engine.beam_state
    assert bs.kernels and bs.table is not None and bs.graph is not None
    assert int(bs.dec.pos.max()) == ids.shape[1] + n_new - 1 == bs.table.shape[1] * 128 - 1
    model.engine.beam_state = None
    orig = G.beam_state

    def physical(*a):
        st = orig(*a)
        st.table = None                                                   # attention reads row b; beam_reorder moves rows
        return st

    monkeypatch.setattr(G, "beam_state", physical)
    monkeypatch.setenv("ODB_CUDA_GRAPH", "0")
    ref = model.generate(ids, **kw)
    model.engine.beam_state = None
    assert torch.equal(got.sequences, ref.sequences)
    assert torch.equal(got.sequences_scores, ref.sequences_scores)


@pytest.mark.parametrize("shape", ["150m_layer", "1b_gqa_layer"])
def test_scores_match_score(shape):
    """score() is an independent oracle: each hypothesis's score is the sum of its generated tokens' log-probs over
    generated_len ** length_penalty.  The histories cross 128-key chunks, so a wrong chunk table shows here."""
    model = LlamaForCausalLM(_layer_cfg(shape), device="cuda", precision="bf16-mixed", seed=7)
    ids, mask = _prompts()
    P, n_new, nb, lp = ids.shape[1], 130, 4, 1.5
    got = model.generate(ids, attention_mask=mask, max_new_tokens=n_new, num_beams=nb, num_return_sequences=nb, eos_token_id=[],
                         length_penalty=lp, return_dict_in_generate=True)
    full_mask = torch.cat([mask.repeat_interleave(nb, 0), torch.ones(ids.shape[0] * nb, n_new, dtype=mask.dtype, device="cuda")], 1)
    lp_tok = model.score(got.sequences, attention_mask=full_mask).logprobs[:, P:]
    want = lp_tok.sum(dim=1) / n_new ** lp
    rel = ((got.sequences_scores - want).abs() / want.abs()).max().item()
    assert rel < 2e-2, rel


def _our_kernel_names() -> set[str]:
    names = set()
    for src in CSRC.glob("*.cu"):
        names |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(", src.read_text()))
    return names


def test_beam_step_launches_only_our_kernels():
    _in_fresh_process("_beam_step_launches_only_our_kernels")


def _beam_step_launches_only_our_kernels():
    model = LlamaForCausalLM(_layer_cfg("1b_gqa_layer"), device="cuda", precision="bf16-mixed", seed=0)
    B, nb, n_new = 2, 4, 8
    bs = beam_state(model, B, nb, DK.beams_to_keep(nb, 1), n_new, 256)
    bs.dec.set_controls(False, 1.0, 0, 1.0, 0, 0, [2])
    bs.reset(0)
    ids = torch.randint(3, V, (B, 128), device="cuda")
    beam_prefill(model, bs, ids, torch.full((B,), 128, dtype=torch.int32, device="cuda"))
    beam_select(bs, 1.0, 0)
    beam_step(model, bs, 1.0, 0, graph=False)
    torch.cuda.synchronize()
    ours = _our_kernel_names()
    assert {"beam_topk_kernel", "beam_step_kernel", "beam_reorder_kernel", "decode_attn_kernel"} <= ours
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        beam_step(model, bs, 1.0, 0, graph=False)
        torch.cuda.synchronize()
    gpu_events = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert any("beam_reorder_kernel" in n for n in gpu_events)
    foreign = [n for n in gpu_events if not any(re.search(rf"\b{k}\b", n) for k in ours)]
    assert not foreign, foreign


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


def test_beam_search_does_not_disturb_training_or_decode_state():
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
    greedy = a.generate(batches[0][:2, :50], max_new_tokens=10)
    dst = a.engine.decode_state
    dec_before = dst.kv.clone()
    ws_before = dict(a.engine._ws)
    state_before = [t.clone() for t in (a.arena.master, a.arena.grad, a.arena.shadow)]
    a.generate(batches[0][:2, :50], max_new_tokens=30, num_beams=4, num_return_sequences=2)
    torch.cuda.synchronize()
    assert a.engine.decode_state is dst and torch.equal(dst.kv, dec_before)
    assert a.engine._graphs[key]["graph"] is g_obj
    assert a.engine._ws == ws_before
    for before, now in zip(state_before, (a.arena.master, a.arena.grad, a.arena.shadow)):
        assert torch.equal(before, now)
    assert torch.equal(a.generate(batches[0][:2, :50], max_new_tokens=10), greedy)
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
