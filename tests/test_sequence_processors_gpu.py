"""``sequence_bias``, ``bad_words_ids``, ``min_length`` and ``min_p`` on an H100: the sampler and beam-selection kernels
against ``process_logits_reference`` / ``beam_step_reference`` with a sequence table, the sampling law with a bias and
min-p, the acceptance law with min-p, graph replay across table contents, the launched kernels, and properties of
``generate`` on a 150m-shaped model."""
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
from scipy import stats

from opendiloco_b200 import _lib
from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.generation import decode_state, prefill, step
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import decode as DK

pytestmark = pytest.mark.gpu

CSRC = Path(__file__).resolve().parent.parent / "opendiloco_b200" / "csrc"
ALPHA = 1e-4


def _table(entries, device="cuda"):
    t = DK.SeqTable(device)
    t.set(entries)
    return t


def _entries(V, h, g, n_bias=40, n_ban=30):
    """Table entries planted on the histories h [rows, S] (lengths L): suffix matches of lengths 1..5, one sequence longer
    than a history, one equal to a whole history plus a token, several biases on one token, and random misses."""
    bias, ban = {}, []
    rows = h.shape[0]
    for i in range(n_bias):
        r = i % rows
        k = 1 + i % 5
        tail = h[r, -(k - 1):].tolist() if k > 1 else []
        bias[tuple(tail) + (int(torch.randint(0, V, (1,), generator=g)),)] = float(torch.randn((), generator=g) * 4)
    bias[(V - 1,)] = 2.5
    bias[(int(h[0, -1]), V - 1)] = -1.25                                     # a second bias on V - 1
    bias[tuple(h[1].tolist()) + (3,)] = 7.0                                  # longer than the history: never matches
    for i in range(n_ban):
        r = i % rows
        k = 1 + i % 4
        tail = h[r, -(k - 1):].tolist() if k > 1 else []
        ban.append(tail + [int(torch.randint(0, V, (1,), generator=g))])
    ban.append([0])
    return DK.sequence_entries(bias, ban, [], V)


# ------------------------------------------------------------------------------------------------ sampler, greedy
@pytest.mark.parametrize("V", [1000, 32000, DK.MAX_SAMPLE_VOCAB])
@pytest.mark.parametrize("penalty,min_len", [(1.0, 0), (1.4, 0), (1.0, 40), (0.7, 40)])
def test_sampler_greedy_matches_reference(V, penalty, min_len):
    g = torch.Generator().manual_seed(V + int(penalty * 10) + min_len)
    B, S = 8, 32
    hist = torch.randint(0, V, (B, S), generator=g).int()
    lens = torch.full((B,), S, dtype=torch.int32)
    entries = _entries(V, hist, g)
    logits = (torch.randn(B, V, generator=g) * 2).bfloat16()
    # put the biased and banned tokens near the top so the table decides the argmax
    for ids, _, _ in entries:
        logits[:, ids[-1]] = logits[:, ids[-1]].float().add(6.0).bfloat16()
    eos = [int(hist[0, 3]), 5]
    ictl, fctl = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, eos, "cpu", penalty, 0, 0, min_len, 0.0, len(entries))
    results = []
    for dev in ("cuda", "cpu"):
        pos = (lens - 1).to(dev)
        z = lambda: torch.zeros(B, dtype=torch.int32, device=dev)           # noqa: E731
        out = torch.zeros(B, 4, dtype=torch.int64, device=dev)
        ids = torch.zeros(B, dtype=torch.int64, device=dev)
        scratch = torch.full((B, 2 * ((V + 31) // 32)), -1, dtype=torch.int32, device=dev)
        seq_scratch = torch.zeros(B, V, device=dev)
        DK.sample(logits.to(dev), ictl.to(dev), fctl.to(dev), pos, z(), z(), out, ids, hist.to(dev).clone(), scratch,
                  _table(entries, dev), seq_scratch)
        results.append(ids.cpu())
        if dev == "cuda":
            assert int(torch.count_nonzero(seq_scratch)) == 0                 # the kernel leaves the bias rows zero
    assert torch.equal(results[0], results[1])
    plain = logits.float().argmax(-1)
    assert not torch.equal(results[0], plain)


# ------------------------------------------------------------------------------------------------ sampling law
def test_sampling_law_with_bias_and_min_p():
    V, T, k, p, min_p = 32000, 0.9, 0, 0.95, 0.05
    g = torch.Generator().manual_seed(1)
    x = torch.randn(V, generator=g) * 0.5
    head = torch.randperm(V, generator=g)[:40]
    x[head] = torch.linspace(4.0, 1.0, 40)
    S = 16
    h = torch.randint(0, V, (S,), generator=g).int()
    entries = DK.sequence_entries({(int(head[0]),): -3.0, (int(h[-1]), int(head[5])): 2.0, (int(head[10]),): 1.5,
                                   (int(h[-2]), int(h[-1]), int(head[10])): 0.75}, [[int(head[1])]], [], V)
    xb = x.bfloat16()
    proc = DK.process_logits_reference(xb.float()[None], h[None], torch.tensor([S]), torch.zeros(1), 1.0, 0, 0, [], entries)[0]
    want = torch.softmax(DK.warp_logits(proc.double()[None], T, k, p, min_p)[0], -1)
    raw = torch.softmax(DK.warp_logits(xb.double()[None], T, k, p, min_p)[0], -1)
    assert (want - raw).abs().sum() > 0.2
    B, reps = 16384, 8
    logits = xb.cuda()[None].expand(B, V)
    hist = h[None].repeat(B, 1).cuda()
    tab = _table(entries)
    seq_scratch = torch.zeros(B, V, device="cuda")
    counts = torch.zeros(V, dtype=torch.int64)
    for rep in range(reps):
        ictl, fctl = DK.make_controls(True, T, k, p, 1000 + rep, 0, [], "cuda", 1.0, 0, 0, 0, min_p, len(entries))
        pos = torch.full((B,), S - 1, dtype=torch.int32, device="cuda")
        z = lambda: torch.zeros(B, dtype=torch.int32, device="cuda")        # noqa: E731
        out = torch.zeros(B, 1, dtype=torch.int64, device="cuda")
        ids = torch.zeros(B, dtype=torch.int64, device="cuda")
        scratch = torch.empty(B, 2 * ((V + 31) // 32), dtype=torch.int32, device="cuda")
        DK.sample(logits, ictl, fctl, pos, z(), z(), out, ids, hist.clone(), scratch, tab, seq_scratch)
        counts += torch.bincount(ids.cpu(), minlength=V)
    N = B * reps
    # tokens within fp32 rounding of a cut: neither kept nor removed for sure
    lo = torch.softmax(DK.warp_logits(proc.double()[None], T, k, min(1.0, p + 1e-3), min_p * (1 - 1e-4))[0], -1)
    edge = (want == 0) & (lo > 0)
    assert int(counts[(want == 0) & ~edge].sum()) == 0
    exp = (want * (N - int(counts[edge].sum()))).numpy()
    obs = counts.masked_fill(edge, 0).numpy().astype(np.float64)
    keep = exp >= 5
    o = np.append(obs[keep], obs[~keep].sum())
    e = np.append(exp[keep], exp[~keep].sum())
    if e[-1] < 5:
        o, e = o[:-1], e[:-1]
        e = e * o.sum() / e.sum()
    assert stats.chisquare(o, e).pvalue > ALPHA


@pytest.mark.parametrize("mode", ["draft", "point_mass"])
def test_accept_law_with_min_p(mode):
    """One acceptance slot (K = 1) with min-p on p and q: the emitted first token follows the fp64 law of p after the
    warpers (speculative sampling is exact), and min-p removes what it must."""
    V, T, min_p = 32000, 1.0, 0.02
    g = torch.Generator().manual_seed(3)
    pl = torch.randn(2, V, generator=g) * 0.5
    pl[:, :30] += torch.linspace(4, 1, 30)
    ql = pl[:1] + torch.randn(1, V, generator=g) * 0.7
    pb, qb = pl.bfloat16(), ql.bfloat16()
    p0 = torch.softmax(DK.warp_logits(pb[:1].double(), T, 0, 1.0, min_p)[0], -1)
    q0 = torch.softmax(DK.warp_logits(qb.double(), T, 0, 1.0, min_p)[0], -1)
    B, reps = 16384, 6
    counts = torch.zeros(V, dtype=torch.int64)
    d_fixed = 1
    for rep in range(reps):
        ictl, fctl = DK.make_controls(True, T, 0, 1.0, 77 + rep, 0, [], "cuda", min_p=min_p)
        plog = pb.cuda().repeat_interleave(B, 0)                             # slot-major: slot 0 rows, then slot 1 rows
        tok = torch.zeros(2 * B, dtype=torch.int64, device="cuda")
        if mode == "draft":
            qlog = qb.cuda().expand(B, V)
            tok[B:] = torch.multinomial(q0.float().cuda(), B, replacement=True, generator=torch.Generator("cuda").manual_seed(rep))
            cnt = None
        else:
            qlog = None
            tok[B:] = d_fixed
            cnt = torch.ones(B, dtype=torch.int32, device="cuda")
        z = lambda: torch.zeros(B, dtype=torch.int32, device="cuda")        # noqa: E731
        out = torch.zeros(B, 4, dtype=torch.int64, device="cuda")
        stats_ = torch.zeros(B, 2, dtype=torch.int64, device="cuda")
        DK.accept(plog, qlog, ictl, fctl, tok, z(), z(), z(), out, 4, None, stats_, cnt=cnt)
        counts += torch.bincount(out[:, 0].cpu(), minlength=V)
    N = B * reps
    assert int(counts[p0 == 0].sum()) == 0
    exp = (p0 * N).numpy()
    obs = counts.numpy().astype(np.float64)
    keep = exp >= 5
    o = np.append(obs[keep], obs[~keep].sum())
    e = np.append(exp[keep], exp[~keep].sum())
    if e[-1] < 5:
        o, e = o[:-1], e[:-1]
        e = e * o.sum() / e.sum()
    assert stats.chisquare(o, e).pvalue > ALPHA


# ------------------------------------------------------------------------------------------------ beam selection
@pytest.mark.parametrize("penalty", [1.0, 1.8])
@pytest.mark.parametrize("nb", [4, 8])
def test_select_kernels_match_reference(penalty, nb):
    B, M, t, n_eos, V = 4, 40, 20, 2, 32000
    K = DK.beams_to_keep(nb, n_eos)
    rows = B * nb
    g = torch.Generator().manual_seed(nb * 7 + int(penalty))
    S = 64
    prompt = torch.randint(0, 8, (B, S), generator=g).int()
    plens = torch.tensor([5, 64, 30, 1], dtype=torch.int32)
    hist = torch.randint(0, 8, (2, rows, M), generator=g).int()
    hist[:, :, t:] = 0
    hist[:, 2 * nb:3 * nb] = 0
    logits = 3 * torch.randn(rows, V, generator=g)
    logits[:, :8] += 8
    logits[:, 100:108] += 5 + 2 * torch.rand(rows, 8, generator=g)
    logits = logits.bfloat16()
    eos = [100, 3]
    # biases on history tokens (penalised too), on fresh tokens at the top, two on one token, ties of equal biased values
    bias = {(1,): 3.0, (2,): -2.0, (101,): 1.5, (7, 102): 4.0, (0, 7, 102): -1.0, (5,): 0.0, (6,): 0.0,
            (3, 4, 200): 30.0, (4, 201): 25.0}
    bad = [[0], [5, 6], [1, 2, 4]]
    entries = DK.sequence_entries(bias, bad, eos, V)
    logits[:, 200] = logits[:, 201] = logits[:, 200].float().bfloat16()   # equal raw logits: ties after equal bias
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
    ictl, fctl = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, eos, "cpu", penalty, 0, 0, 30, 0.0, len(entries))
    ref = {k: v.clone() for k, v in st.items()}
    DK.beam_step_reference(logits, ictl, nb, K, 1.3, 0, M, **ref, fctl=fctl, prompt=prompt, plens=plens, table=_table(entries, "cpu"))
    plain = {k: v.clone() for k, v in st.items()}
    c0, f0 = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, eos, "cpu", penalty, 0, 0)
    DK.beam_step_reference(logits, c0, nb, K, 1.3, 0, M, **plain, fctl=f0, prompt=prompt, plens=plens)
    assert any(not torch.equal(plain[k], ref[k]) for k in ("ids_next", "parent", "run_score"))
    gpu = {k: v.cuda() for k, v in st.items()}
    nsp = DK.beam_splits(V)
    DK.beam_select(logits.cuda(), ictl.cuda(), nb, K, 1.3, 0, M, **gpu, part_ml=torch.empty(rows, nsp, 2, device="cuda"),
                   cand_v=torch.empty(rows, nsp, 2 * K, device="cuda"),
                   cand_i=torch.empty(rows, nsp, 2 * K, dtype=torch.int32, device="cuda"), fctl=fctl.cuda(), prompt=prompt.cuda(),
                   plens=plens.cuda(), table=_table(entries), slot_i=torch.full((rows, DK.MAX_SEQS), 7, dtype=torch.int32, device="cuda"),
                   slot_v=torch.zeros(rows, DK.MAX_SEQS, 2, device="cuda"))
    torch.cuda.synchronize()
    for k in ("fin_flag", "run_seq", "fin_seq", "unsat", "done", "tstep", "pos", "ids_next", "parent"):
        assert torch.equal(gpu[k].cpu(), ref[k]), k
    for k in ("run_score", "fin_score"):
        assert torch.allclose(gpu[k].cpu(), ref[k], atol=2e-5 * max(1.0, penalty), rtol=1e-6), (k, (gpu[k].cpu() - ref[k]).abs().max())


# ------------------------------------------------------------------------------------------------ generate, 150m
@pytest.fixture(scope="module")
def model_150m():
    cfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=12, num_attention_heads=16, vocab_size=32000)
    return LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=11)


def _batch(V, B=4, P=48, seed=0):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, V, (B, P), generator=g)
    mask = torch.ones_like(ids)
    mask[1, :10] = 0
    mask[3, :30] = 0
    return ids.cuda(), mask.cuda()


@pytest.mark.parametrize("fp8_kv", [False, True])
@pytest.mark.parametrize("mode", ["greedy", "sample", "multi", "beam"])
def test_bad_words_never_occur_and_min_length_holds(model_150m, mode, fp8_kv):
    V, n_new = 32000, 256
    ids, mask = _batch(V)
    free = model_150m.generate(ids, attention_mask=mask, max_new_tokens=64, eos_token_id=[])[:, ids.shape[1]:].tolist()
    # ban what the unconstrained run does: its first token, a pair and a triple of its continuation
    bad = [[free[0][0]], free[1][3:5], free[2][6:9], [free[3][10]]]
    eos = free[0][2]
    kw = dict(attention_mask=mask, max_new_tokens=n_new, eos_token_id=[eos], pad_token_id=0, bad_words_ids=bad,
              min_length=ids.shape[1] + 100, fp8_kv_cache=fp8_kv,
              sequence_bias={(free[0][1],): -2.0, (free[1][0], free[1][1]): 1.0})
    if mode == "sample":
        kw.update(do_sample=True, seed=3, top_k=0, min_p=0.02)
    elif mode == "multi":
        kw.update(do_sample=True, seed=4, num_return_sequences=3)
    elif mode == "beam":
        kw.update(num_beams=4, num_return_sequences=2)
    out = model_150m.generate(ids, **kw)
    R = out.shape[0] // ids.shape[0]
    for r, row in enumerate(out.tolist()):
        b = r // R
        plen = int(mask[b].sum())
        new = row[ids.shape[1]:]
        if eos in new:
            new = new[:new.index(eos) + 1]
            # min_length counts the real prompt: no EOS while the history is shorter than min_length
            assert plen + new.index(eos) >= ids.shape[1] + 100, (plen, new.index(eos))
        hist = row[ids.shape[1] - plen:ids.shape[1]] + new
        for w in bad:                                # no generated token completes a bad word
            k = len(w)
            assert not any(hist[i - k + 1:i + 1] == w for i in range(max(plen, k - 1), len(hist))), (w, r)


def test_graph_equals_eager_and_tables_do_not_recapture(monkeypatch):
    cfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=1, num_attention_heads=16, vocab_size=32000)
    model = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=4)
    ids, mask = _batch(32000)
    free = model.generate(ids, attention_mask=mask, max_new_tokens=16, eos_token_id=[])[:, ids.shape[1]:].tolist()
    settings = [dict(bad_words_ids=[[free[0][0]]]),
                dict(bad_words_ids=[free[1][2:4], [free[2][0]]], sequence_bias={(free[0][1],): -5.0}, min_length=60),
                dict(sequence_bias={tuple(free[3][:3]): 8.0, (17,): 3.0}, repetition_penalty=1.3, min_p=0.1, do_sample=True),
                dict(bad_words_ids=[[t, 5] for t in range(3, 1000)], min_length=70)]
    for num_beams in (1, 4):
        kw = dict(attention_mask=mask, max_new_tokens=40, num_beams=num_beams, eos_token_id=[17, 99], return_dict_in_generate=True)
        monkeypatch.setenv("ODB_CUDA_GRAPH", "1")
        graphed, graph = [], None
        for s in settings:
            s = dict(s)
            if num_beams > 1:
                s.pop("do_sample", None)
            graphed.append(model.generate(ids, **kw, **s))
            st = model.engine.beam_state if num_beams > 1 else model.engine.decode_state
            assert st.graph is not None and (graph is None or st.graph is graph)
            graph = st.graph
        monkeypatch.setenv("ODB_CUDA_GRAPH", "0")
        for s, got in zip(settings, graphed):
            s = dict(s)
            if num_beams > 1:
                s.pop("do_sample", None)
            eager = model.generate(ids, **kw, **s)
            assert torch.equal(got.sequences, eager.sequences)
            if num_beams > 1:
                assert torch.equal(got.sequences_scores, eager.sequences_scores)


# ------------------------------------------------------------------------------------------------ launches
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


def test_steps_launch_only_our_kernels_and_defaults_launch_as_before():
    _in_fresh_process("_launches")


def _launches():
    cfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=1, num_attention_heads=16, vocab_size=32000)
    model = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=0)
    ours = _our_kernel_names()
    ids = torch.randint(3, cfg.vocab_size, (4, 128), device="cuda")
    st = decode_state(model, 4, 256)
    st.set_controls(True, 0.8, 40, 0.9, 0, 0, [2], 1.2, 3, 4, min_length=200, min_p=0.05,
                    entries=DK.sequence_entries({(5,): 1.0, (6, 7): -1.0}, [[9, 10]], [2], cfg.vocab_size))
    prefill(model, st, ids, torch.full((4,), 128, dtype=torch.int32, device="cuda"))
    step(model, st, graph=False)
    names = _gpu_kernels(lambda: step(model, st, graph=False))
    assert any("sample_kernel" in n for n in names)
    assert not [n for n in names if not any(re.search(rf"\b{k}\b", n) for k in ours)]
    # the defaults launch what they launched before: the same count as an explicit all-defaults call (after a first call,
    # which warms up and captures the step graph that both replay)
    x = torch.randint(3, cfg.vocab_size, (2, 40), device="cuda")
    for kw in (dict(), dict(num_beams=4), dict(do_sample=True, num_return_sequences=2)):
        model.generate(x, max_new_tokens=12, **kw)
        c0 = _lib.launch_count()
        a = model.generate(x, max_new_tokens=12, **kw)
        c1 = _lib.launch_count()
        b = model.generate(x, max_new_tokens=12, sequence_bias=None, bad_words_ids=None, min_length=0, min_p=None, **kw)
        c2 = _lib.launch_count()
        assert torch.equal(a, b) and c1 - c0 == c2 - c1, (kw, c1 - c0, c2 - c1)


def _in_fresh_process(fn: str) -> None:
    here = Path(__file__).resolve()
    code = f"import sys; sys.path[:0] = [{str(here.parents[1])!r}, {str(here.parent)!r}]; import {here.stem}; {here.stem}.{fn}()"
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=here.parents[1], timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-6000:]
