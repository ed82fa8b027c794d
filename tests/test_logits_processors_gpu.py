"""Logits processors on an H100: the sampler kernel and the beam-selection kernels against ``process_logits_reference``
and ``beam_step_reference``, the sampling law on processed logits, the whole program against the references, graph
replay, and properties of ``generate`` on a 150m-shaped model."""
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from scipy import stats

from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.generation import beam_prefill, beam_select, beam_state, beam_step, decode_state, prefill, step
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import decode as DK

pytestmark = pytest.mark.gpu

CSRC = Path(__file__).resolve().parent.parent / "opendiloco_b200" / "csrc"
ALPHA = 1e-4


# ------------------------------------------------------------------------------------------------ sampler, greedy
def _histories(V, S, g):
    """Eight rows of histories [8, S] with their lengths: one token; duplicates with tokens 0 and V - 1; S tokens (a full
    cache); overlapping n-gram matches; a match at position 0; a history shorter than n; two rows for min_new_tokens."""
    h = torch.randint(0, V, (8, S), generator=g)
    rows = [[V - 1], [0, V - 1, 5, 0, V - 1, 5, 0, V - 1], None, [7] * 9, [9, 4, 2, 9, 4, 11, 9, 4], [3, V - 2],
            [1, 2, 3, 1, 2], [1, 2, 3, 1, 2]]
    lens = []
    for r, toks in enumerate(rows):
        if toks is None:
            h[r] = torch.randint(0, 12, (S,), generator=g)                  # small alphabet: many matches over S tokens
            lens.append(S)
        else:
            h[r, :len(toks)] = torch.tensor(toks)
            lens.append(len(toks))
    return h.int(), torch.tensor(lens, dtype=torch.int32)


def _run_sampler(logits, ictl, fctl, hist, lens, gen):
    """One sample() call on CUDA (kernel) or CPU (reference); returns (tokens, history after the append)."""
    dev = logits.device
    B, V = logits.shape
    pos = (lens - 1).to(dev)
    gen = gen.to(dev).clone()
    fin = torch.zeros(B, dtype=torch.int32, device=dev)
    out = torch.zeros(B, 4, dtype=torch.int64, device=dev)
    ids = torch.zeros(B, dtype=torch.int64, device=dev)
    h = hist.to(dev).clone()
    scratch = torch.full((B, 2 * ((V + 31) // 32)), -1, dtype=torch.int32, device=dev)      # stale bits must be cleared
    DK.sample(logits, ictl.to(dev), fctl.to(dev), pos, gen, fin, out, ids, h, scratch)
    return ids.cpu(), h.cpu()


@pytest.mark.parametrize("V", [1000, 32000, DK.MAX_SAMPLE_VOCAB])
@pytest.mark.parametrize("penalty,n,m", [(1.3, 0, 0), (0.7, 0, 0), (1.0, 1, 0), (1.0, 2, 0), (1.0, 3, 0), (1.0, 0, 4),
                                         (1.8, 3, 4)])
def test_sampler_greedy_matches_reference(V, penalty, n, m):
    S = 2048
    g = torch.Generator().manual_seed(V + n)
    hist, lens = _histories(V, S, g)
    logits = torch.randn(8, V, generator=g) * 2 + 6
    eos = [int(logits[6].argmax()), int(logits[7].argmax())]
    gen = torch.tensor([0, 1, 2, 3, 4, 5, m - 1, m]).clamp(min=0).int()     # rows 6, 7: the min_new_tokens boundary
    ictl, fctl = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, eos, "cpu", penalty, n, m)
    # make the row's argmax a token the processors move: banned or penalised (p > 1) on top, boosted (p < 1) just below
    proc = DK.process_logits_reference(logits, hist, lens, gen, penalty, n, m, eos)
    for r in range(8):
        moved = (proc[r] != logits[r]).nonzero().flatten()
        if len(moved):
            t, top = int(moved[0]), float(logits[r].max())
            logits[r, t] = top - 0.5 if penalty < 1 and proc[r, t] > float("-inf") else top + 1
    logits = logits.bfloat16()
    got, gh = _run_sampler(logits.cuda(), ictl, fctl, hist, lens, gen)
    ref, rh = _run_sampler(logits, ictl, fctl, hist, lens, gen)
    assert torch.equal(got, ref), (got, ref)
    assert torch.equal(gh, rh)
    assert int(gh[0, 1]) == int(got[0]) and torch.equal(gh[2], hist[2])    # appended at pos + 1; none past a full cache
    assert (ref != logits.float().argmax(-1)).sum() >= 3                   # the processors changed the rows they touch
    if m > 0:
        assert int(got[6]) != eos[0]                                       # gen = m - 1: EOS banned
        if penalty == 1.0 and n == 0:
            assert int(got[7]) == eos[1]                                   # gen = m: EOS allowed again


def test_sampler_all_inf_rows():
    """Every token banned: greedy emits 0, sampling its processed argmax (0 as well)."""
    V = 64
    hist = torch.arange(V, dtype=torch.int32)[None, :].repeat(2, 1)
    lens = torch.full((2,), V, dtype=torch.int32)
    logits = torch.randn(2, V, generator=torch.Generator().manual_seed(0)).bfloat16().cuda()
    for do_sample in (False, True):
        ictl, fctl = DK.make_controls(do_sample, 1.0, 0, 1.0, 0, 0, [], "cpu", 1.0, 1, 0)
        got, _ = _run_sampler(logits, ictl, fctl, hist, lens, torch.zeros(2, dtype=torch.int32))
        assert got.tolist() == [0, 0]


# ------------------------------------------------------------------------------------------------ sampling law
def _law(x64, T, k, p):
    """fp64 law of the sampler on processed logits x64 [V]: HF's warpers (ties kept) then softmax."""
    w = DK.warp_logits(x64[None], T, k, p)[0]
    return torch.softmax(w, -1)


LAW_CASES = {
    # name: (V, temperature, top_k, top_p, penalty, n, head) -- the history holds the head of the row, logits head .. head - 2
    "penalty_across_top_k": (32000, 1.0, 12, 1.0, 2.5, 0, 3.0),
    "penalty_across_top_p": (32000, 0.9, 0, 0.7, 3.0, 0, 10.0),
    "boost_into_top_k": (1000, 1.0, 8, 1.0, 0.4, 0, 3.0),
    "ban_on_segment_edges": (DK.MAX_SAMPLE_VOCAB, 1.2, 0, 1.0, 1.0, 1, 10.0),
    "all_three_warpers": (32000, 0.8, 40, 0.9, 1.5, 2, 3.0),
}


@pytest.mark.parametrize("case", list(LAW_CASES))
def test_sampling_law_on_processed_logits(case):
    V, T, k, p, pen, n, head = LAW_CASES[case]
    g = torch.Generator().manual_seed(len(case))
    x = torch.randn(V, generator=g) * 0.5
    per = (V + 1023) // 1024
    if case == "ban_on_segment_edges":
        toks = [0, per - 1, per, 5 * per - 1, 5 * per, V - 1, V - 2]
    else:
        toks = torch.randperm(V, generator=g)[:16].tolist()
    S = 32
    h = torch.tensor((toks * S)[:S], dtype=torch.int32)
    L = len(toks)
    x[torch.tensor(toks)] = torch.linspace(head, head - 2, L)               # the history holds the head of the row
    x[torch.randperm(V, generator=g)[:20]] += 2.0                           # and a rival head outside it
    xb = x.bfloat16()
    ictl, fctl = DK.make_controls(True, T, k, p, 0, 0, [], "cpu", pen, n, 0)
    proc = DK.process_logits_reference(xb.float()[None], h[None], torch.tensor([L]), torch.zeros(1), pen, n, 0, [])[0]
    want = _law(proc.double(), T, k, p)
    raw = _law(xb.double(), T, k, p)
    assert (want - raw).abs().sum() > 0.2                                   # the processors move real mass
    B, reps = 16384, 8
    logits = xb.cuda()[None].expand(B, V)
    hist = h[None].repeat(B, 1).cuda()
    counts = torch.zeros(V, dtype=torch.int64)
    for rep in range(reps):
        ictl, fctl = DK.make_controls(True, T, k, p, 1000 + rep, 0, [], "cuda", pen, n, 0)
        pos = torch.full((B,), L - 1, dtype=torch.int32, device="cuda")
        z = lambda: torch.zeros(B, dtype=torch.int32, device="cuda")        # noqa: E731
        out = torch.zeros(B, 1, dtype=torch.int64, device="cuda")
        ids = torch.zeros(B, dtype=torch.int64, device="cuda")
        scratch = torch.empty(B, 2 * ((V + 31) // 32), dtype=torch.int32, device="cuda")
        DK.sample(logits, ictl, fctl, pos, z(), z(), out, ids, hist.clone(), scratch)
        counts += torch.bincount(ids.cpu(), minlength=V)
    N = B * reps
    # tokens at the top-p cut within fp32 rounding of the kernel's bisection: neither kept nor removed for sure
    edge = (want == 0) & (_law(proc.double(), T, k, min(1.0, p + 1e-3)) > 0)
    assert int(counts[(want == 0) & ~edge].sum()) == 0                       # removed and banned tokens are never drawn
    exp = (want * (N - int(counts[edge].sum()))).numpy()
    obs = counts.masked_fill(edge, 0).numpy().astype(np.float64)
    keep = exp >= 5
    o = np.append(obs[keep], obs[~keep].sum())
    e = np.append(exp[keep], exp[~keep].sum())
    if e[-1] < 5:
        o, e = o[:-1], e[:-1]
        e = e * o.sum() / e.sum()
    assert stats.chisquare(o, e).pvalue > ALPHA


# ------------------------------------------------------------------------------------------------ beam selection
V_BEAM = 32000


@pytest.mark.parametrize("penalty", [0.5, 2.0])
@pytest.mark.parametrize("n", [0, 2, 3])
@pytest.mark.parametrize("nb", [4, 8])
def test_select_kernels_match_reference(penalty, n, nb):
    B, M, t, n_eos = 4, 40, 20, 2
    V = V_BEAM
    K = DK.beams_to_keep(nb, n_eos)
    rows = B * nb
    g = torch.Generator().manual_seed(nb * 10 + n)
    S = 64
    prompt = torch.randint(0, 8, (B, S), generator=g).int()                # small alphabet: n-gram matches
    plens = torch.tensor([5, 64, 30, 1], dtype=torch.int32)
    hist = torch.randint(0, 8, (2, rows, M), generator=g).int()
    hist[:, :, t:] = 0
    hist[:, 2 * nb:3 * nb] = 0                                              # prompt 2 is at step 0: no running history yet
    logits = 3 * torch.randn(rows, V, generator=g)
    logits[:, :8] += 8                                                      # history tokens at the top, close to others
    logits[:, 100:108] += 5 + 2 * torch.rand(rows, 8, generator=g)
    logits = logits.bfloat16()
    eos = [100, 3]
    run_score = -4 * torch.rand(rows, generator=g)
    fin_flag = (torch.rand(rows, generator=g) < 0.5).int()
    fin_score = torch.where(fin_flag.bool(), -3 * torch.rand(rows, generator=g), torch.full((rows,), DK.NEG))
    fin_seq = hist.flip(1).contiguous()
    fin_seq[:, 2 * nb:3 * nb] = 0
    st = dict(run_score=run_score, fin_score=fin_score, fin_flag=fin_flag, run_seq=hist.clone(), fin_seq=fin_seq,
              unsat=torch.ones(B, dtype=torch.int32), done=torch.zeros(B, dtype=torch.int32),
              tstep=torch.tensor([t, t, 0, t], dtype=torch.int32),
              pos=torch.randint(100, 200, (B,), generator=g).int().repeat_interleave(nb),
              ids_next=torch.zeros(rows, dtype=torch.int64), parent=torch.zeros(rows, dtype=torch.int32))
    st["done"][1] = 1
    ictl, fctl = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, eos, "cpu", penalty, n, 25)
    ref = {k: v.clone() for k, v in st.items()}
    DK.beam_step_reference(logits, ictl, nb, K, 1.3, 0, M, **ref, fctl=fctl, prompt=prompt, plens=plens)
    plain = {k: v.clone() for k, v in st.items()}
    DK.beam_step_reference(logits, ictl, nb, K, 1.3, 0, M, **plain)
    assert any(not torch.equal(plain[k], ref[k]) for k in ("ids_next", "parent", "run_score", "fin_score"))   # processors matter
    gpu = {k: v.cuda() for k, v in st.items()}
    nsp = DK.beam_splits(V)
    part_ml = torch.empty(rows, nsp, 2, device="cuda")
    cand_v = torch.empty(rows, nsp, 2 * K, device="cuda")
    cand_i = torch.empty(rows, nsp, 2 * K, dtype=torch.int32, device="cuda")
    DK.beam_select(logits.cuda(), ictl.cuda(), nb, K, 1.3, 0, M, **gpu, part_ml=part_ml, cand_v=cand_v, cand_i=cand_i,
                   fctl=fctl.cuda(), prompt=prompt.cuda(), plens=plens.cuda())
    torch.cuda.synchronize()
    for k in ("fin_flag", "run_seq", "fin_seq", "unsat", "done", "tstep", "pos", "ids_next", "parent"):
        assert torch.equal(gpu[k].cpu(), ref[k]), k
    # The two paths round the row's log-sum-exp differently (kernel: split partials; reference: log_softmax); with the
    # boosted head the lse is about 20 here, where a few fp32 ulps are 1e-5, and the penalty scales that error by p.
    for k in ("run_score", "fin_score"):
        assert torch.allclose(gpu[k].cpu(), ref[k], atol=2e-5 * max(1.0, penalty), rtol=1e-6), (k, (gpu[k].cpu() - ref[k]).abs().max())


def test_select_kernels_tiny_vocabulary_inf_ties():
    """n = 1 bans every history token of a 1024-token vocabulary but token 0: the -inf candidates go by beam * V + token."""
    B, nb, M, t, V = 2, 4, 8, 3, 1024
    K = DK.beams_to_keep(nb, 1)
    rows = B * nb
    g = torch.Generator().manual_seed(0)
    prompt = torch.arange(V, dtype=torch.int32)[None].repeat(B, 1)
    prompt[:, 0] = V - 1                                                    # token 0 stays allowed: nb < K finite candidates
    plens = torch.full((B,), V, dtype=torch.int32)
    hist = torch.full((2, rows, M), 5, dtype=torch.int32)
    logits = torch.randn(rows, V, generator=g).bfloat16()
    run_score = torch.zeros(B, nb)
    run_score[:, 1:] = float("-inf")                                        # one finite candidate per prompt, then -inf ties
    st = dict(run_score=run_score.flatten(), fin_score=torch.full((rows,), DK.NEG), fin_flag=torch.zeros(rows, dtype=torch.int32),
              run_seq=hist.clone(), fin_seq=hist.clone(), unsat=torch.ones(B, dtype=torch.int32), done=torch.zeros(B, dtype=torch.int32),
              tstep=torch.full((B,), t, dtype=torch.int32), pos=torch.full((rows,), 50, dtype=torch.int32),
              ids_next=torch.zeros(rows, dtype=torch.int64), parent=torch.zeros(rows, dtype=torch.int32))
    ictl, fctl = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, [9], "cpu", 1.0, 1, 0)
    ref = {k: v.clone() for k, v in st.items()}
    DK.beam_step_reference(logits, ictl, nb, K, 1.0, 0, M, **ref, fctl=fctl, prompt=prompt, plens=plens)
    assert bool(torch.isinf(ref["run_score"]).any()) and ref["ids_next"].view(B, nb)[:, 1:].tolist() == [[1, 2, 3]] * B
    gpu = {k: v.cuda() for k, v in st.items()}
    nsp = DK.beam_splits(V)
    DK.beam_select(logits.cuda(), ictl.cuda(), nb, K, 1.0, 0, M, **gpu, part_ml=torch.empty(rows, nsp, 2, device="cuda"),
                   cand_v=torch.empty(rows, nsp, 2 * K, device="cuda"), cand_i=torch.empty(rows, nsp, 2 * K, dtype=torch.int32, device="cuda"),
                   fctl=fctl.cuda(), prompt=prompt.cuda(), plens=plens.cuda())
    torch.cuda.synchronize()
    for k in ("run_seq", "ids_next", "parent", "fin_flag"):
        assert torch.equal(gpu[k].cpu(), ref[k]), k
    assert torch.equal(gpu["run_score"].cpu(), ref["run_score"])


# ------------------------------------------------------------------------------------------------ whole program
def _layer_cfg(shape):
    if shape == "150m_layer":
        return LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=1, num_attention_heads=16, vocab_size=V_BEAM)
    return LlamaConfig(hidden_size=2048, intermediate_size=5632, num_hidden_layers=1, num_attention_heads=32, num_key_value_heads=4,
                       vocab_size=V_BEAM)


def _prompts(n=3, P=150, seed=5, V=V_BEAM):
    ids = torch.randint(3, V, (n, P), generator=torch.Generator().manual_seed(seed)).cuda()
    mask = torch.ones_like(ids)
    mask[1, :40] = 0
    mask[2, :P - 1] = 0
    return ids, mask


PROC = dict(repetition_penalty=1.3, no_repeat_ngram_size=3, min_new_tokens=5)


@pytest.mark.parametrize("shape", ["150m_layer", "1b_gqa_layer"])
def test_kernels_equal_reference_program(shape, monkeypatch):
    model = LlamaForCausalLM(_layer_cfg(shape), device="cuda", precision="bf16-mixed", seed=6)
    with torch.no_grad():
        dict(model.named_parameters())["model.layers.0.self_attn.o_proj.weight"].zero_()
    model.arena.sync_shadow()
    ids, mask = _prompts()
    P = ids.shape[1]
    first = model.generate(ids, attention_mask=mask, max_new_tokens=4, eos_token_id=[])
    eos = [int(first[0, P + 1]), int(first[1, P + 2]), 99]                  # tokens the rows emit early: min_new_tokens bites
    greedy = model.generate(ids, attention_mask=mask, max_new_tokens=40, eos_token_id=eos, **PROC)
    beams = model.generate(ids, attention_mask=mask, max_new_tokens=40, num_beams=4, num_return_sequences=2, eos_token_id=eos,
                           return_dict_in_generate=True, **PROC)
    assert model.engine.decode_state.kernels and model.engine.beam_state.kernels
    plain = model.generate(ids, attention_mask=mask, max_new_tokens=40, eos_token_id=eos)
    assert not torch.equal(greedy, plain)
    model.engine.decode_state = model.engine.beam_state = None
    orig = DK._lib.has_symbol
    with monkeypatch.context() as m:
        m.setattr(DK._lib, "has_symbol", lambda name: name != "odb_dec_sample" and orig(name))   # every decode op on the references
        ref_greedy = model.generate(ids, attention_mask=mask, max_new_tokens=40, eos_token_id=eos, **PROC)
        ref_beams = model.generate(ids, attention_mask=mask, max_new_tokens=40, num_beams=4, num_return_sequences=2, eos_token_id=eos,
                                   return_dict_in_generate=True, **PROC)
        assert not model.engine.decode_state.kernels and not model.engine.beam_state.kernels
    model.engine.decode_state = model.engine.beam_state = None
    assert torch.equal(greedy, ref_greedy)
    assert torch.equal(beams.sequences, ref_beams.sequences)
    assert torch.allclose(beams.sequences_scores, ref_beams.sequences_scores, atol=1e-5, rtol=0)


@pytest.mark.parametrize("num_beams", [1, 4])
def test_graph_equals_eager_and_values_do_not_recapture(num_beams, monkeypatch):
    model = LlamaForCausalLM(_layer_cfg("150m_layer"), device="cuda", precision="bf16-mixed", seed=4)
    ids, mask = _prompts()
    kw = dict(attention_mask=mask, max_new_tokens=40, num_beams=num_beams, eos_token_id=[17, 99, 1000], return_dict_in_generate=True)
    settings = [dict(), PROC, dict(repetition_penalty=0.8, no_repeat_ngram_size=1), dict(min_new_tokens=30, no_repeat_ngram_size=2)]
    monkeypatch.setenv("ODB_CUDA_GRAPH", "1")
    graphed, graph = [], None
    for s in settings:
        graphed.append(model.generate(ids, **kw, **s))
        st = model.engine.beam_state if num_beams > 1 else model.engine.decode_state
        assert st.graph is not None and (graph is None or st.graph is graph)       # one capture serves every setting
        graph = st.graph
    monkeypatch.setenv("ODB_CUDA_GRAPH", "0")
    for s, got in zip(settings, graphed):
        eager = model.generate(ids, **kw, **s)
        assert torch.equal(got.sequences, eager.sequences)
        if num_beams > 1:
            assert torch.equal(got.sequences_scores, eager.sequences_scores)
    assert not torch.equal(graphed[0].sequences, graphed[1].sequences)


# ------------------------------------------------------------------------------------------------ properties, 150m
@pytest.fixture(scope="module")
def model_150m():
    cfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=12, num_attention_heads=16, vocab_size=32000)
    return LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=11)


def _batch8(V, P=64):
    ids = torch.randint(3, 200, (8, P), generator=torch.Generator().manual_seed(2)).cuda()        # small alphabet: repeats
    mask = torch.ones_like(ids)
    for b in range(8):
        mask[b, :5 * b] = 0
    return ids.masked_fill(mask == 0, 0), mask


def _histories_of(out, ids, mask, eos):
    P = ids.shape[1]
    R = out.shape[0] // ids.shape[0]
    for r in range(out.shape[0]):
        b = r // R
        new = out[r, P:].tolist()
        for i, t in enumerate(new):
            if t in eos:
                new = new[:i + 1]
                break
        yield ids[b][mask[b].bool()].tolist() + new, len(new)


@pytest.mark.parametrize("mode", ["greedy", "sample", "beam"])
def test_no_ngram_occurs_twice(model_150m, mode):
    n = 3
    ids, mask = _batch8(32000)
    kw = {"greedy": {}, "sample": dict(do_sample=True, temperature=0.7, top_k=20, seed=3),
          "beam": dict(num_beams=4, num_return_sequences=2)}[mode]
    eos = [2]
    out = model_150m.generate(ids, attention_mask=mask, max_new_tokens=256, eos_token_id=eos, no_repeat_ngram_size=n, **kw)
    assert model_150m.engine.decode_state.kernels
    for h, _ in _histories_of(out, ids, mask, eos):
        grams = [tuple(h[i:i + n]) for i in range(len(h) - n + 1)]
        assert len(grams) == len(set(grams))
    plain = model_150m.generate(ids, attention_mask=mask, max_new_tokens=256, eos_token_id=eos, **kw)
    repeated = 0
    for h, _ in _histories_of(plain, ids, mask, eos):
        grams = [tuple(h[i:i + n]) for i in range(len(h) - n + 1)]
        repeated += len(grams) - len(set(grams))
    assert repeated > 0                                                          # the unconstrained model does repeat


def test_min_new_tokens_holds_eos_back(model_150m):
    ids, mask = _batch8(32000)
    P, m = ids.shape[1], 40
    free = model_150m.generate(ids, attention_mask=mask, max_new_tokens=256, eos_token_id=[])[:, P:]
    eos = int(torch.mode(free[:, :m].flatten()).values)                          # a token the model emits often, early
    assert (free[:, :m] == eos).any()
    for kw in (dict(), dict(do_sample=True, seed=5, top_k=10), dict(num_beams=4)):
        out = model_150m.generate(ids, attention_mask=mask, max_new_tokens=256, eos_token_id=eos, min_new_tokens=m, **kw)[:, P:]
        assert not (out[:, :m] == eos).any(), kw


def test_greedy_penalty_is_argmax_of_processed_teacher_forced_logits(model_150m):
    ids, mask = _batch8(32000)
    P, n_new, pen = ids.shape[1], 64, 1.3
    out = model_150m.generate(ids, attention_mask=mask, max_new_tokens=n_new, eos_token_id=[], repetition_penalty=pen)
    full_mask = torch.cat([mask, torch.ones(8, n_new, dtype=mask.dtype, device="cuda")], 1)
    logits = model_150m(out, attention_mask=full_mask).logits.float()
    checked = 0
    for b in range(8):
        real = mask[b].bool()
        hist = out[b, :P][real].tolist()
        for j in range(n_new):
            x = logits[b, P - 1 + j][None]
            h = torch.tensor(hist, dtype=torch.int32)[None]
            proc = DK.process_logits_reference(x, h, torch.tensor([len(hist)]), torch.tensor([j]), pen, 0, 0, [])[0]
            top2 = proc.topk(2).values
            tok = int(out[b, P + j])
            if float(top2[0] - top2[1]) > 0.1:                                   # beyond the bf16 noise of teacher forcing
                assert tok == int(proc.argmax()), (b, j)
                checked += 1
            hist.append(tok)
    assert checked > 8 * n_new // 4, checked


# ------------------------------------------------------------------------------------------------ launches and isolation
def _our_kernel_names() -> set[str]:
    names = set()
    for src in CSRC.glob("*.cu"):
        names |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(", src.read_text()))
    return names


def _gpu_kernels(fn):
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_steps_with_processors_launch_only_our_kernels():
    _in_fresh_process("_steps_with_processors_launch_only_our_kernels")


def _steps_with_processors_launch_only_our_kernels():
    cfg = _layer_cfg("1b_gqa_layer")
    model = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=0)
    ours = _our_kernel_names()
    ids = torch.randint(3, cfg.vocab_size, (4, 128), device="cuda")
    st = decode_state(model, 4, 256)
    st.set_controls(True, 0.8, 40, 0.9, 0, 0, [2], 1.2, 3, 4)
    prefill(model, st, ids, torch.full((4,), 128, dtype=torch.int32, device="cuda"))
    step(model, st, graph=False)
    names = _gpu_kernels(lambda: step(model, st, graph=False))
    assert any("sample_kernel" in n for n in names)
    assert not [n for n in names if not any(re.search(rf"\b{k}\b", n) for k in ours)]
    B, nb = 2, 4
    bs = beam_state(model, B, nb, DK.beams_to_keep(nb, 1), 8, 256)
    bs.dec.set_controls(False, 1.0, 0, 1.0, 0, 0, [2], 1.2, 3, 4)
    bs.reset(0)
    bs.prompt[:, :128].copy_(ids[:B])
    bs.plens.fill_(128)
    beam_prefill(model, bs, ids[:B], torch.full((B,), 128, dtype=torch.int32, device="cuda"))
    beam_select(bs, 1.0, 0)
    beam_step(model, bs, 1.0, 0, graph=False)
    names = _gpu_kernels(lambda: beam_step(model, bs, 1.0, 0, graph=False))
    assert any("beam_topk_kernel" in n for n in names)
    assert not [n for n in names if not any(re.search(rf"\b{k}\b", n) for k in ours)]


def test_processors_do_not_disturb_training_or_decode_state():
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
    greedy = a.generate(batches[0][:2, :50], max_new_tokens=10)
    dst = a.engine.decode_state
    dec_before = dst.kv.clone()
    ws_before = dict(a.engine._ws)
    state_before = [t.clone() for t in (a.arena.master, a.arena.grad, a.arena.shadow)]
    a.generate(batches[0][:2, :50], max_new_tokens=30, num_beams=4, num_return_sequences=2, **PROC)
    torch.cuda.synchronize()
    assert a.engine.decode_state is dst and torch.equal(dst.kv, dec_before)
    assert a.engine._graphs[key]["graph"] is g_obj and a.engine._ws == ws_before
    for before, now in zip(state_before, (a.arena.master, a.arena.grad, a.arena.shadow)):
        assert torch.equal(before, now)
    a.generate(batches[0][:2, :50], max_new_tokens=10, **PROC)
    assert torch.equal(a.generate(batches[0][:2, :50], max_new_tokens=10), greedy)
    for x in batches[4:]:
        la.append(a.forward_backward(x, x, 1.0).item())
        lb.append(b.forward_backward(x, x, 1.0).item())
    assert a.engine._graphs[key]["graph"] is g_obj
    for u, v in zip(la, lb):
        assert abs(u - v) <= 1e-5 * abs(v), (la, lb)


def _in_fresh_process(fn: str) -> None:
    """Run ``fn`` of this module in a new Python process and fail with its traceback if it fails.  Used by the tests that
    read kernel names from the CUDA profiler: late in a long pytest process the profiler intermittently records no GPU
    activity at all, while a fresh process records every launch."""
    here = Path(__file__).resolve()
    code = f"import sys; sys.path[:0] = [{str(here.parents[1])!r}, {str(here.parent)!r}]; import {here.stem}; {here.stem}.{fn}()"
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=here.parents[1], timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-6000:]
