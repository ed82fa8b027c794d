"""Prompt lookup decoding on an H100: ``lookup_propose_kernel`` and the point-mass mode of ``accept_kernel``
(csrc/decode_sm90.cu) against the PyTorch references and exact fp64 laws, and ``generate(prompt_lookup_num_tokens=...)``
end to end."""
import json
import os
import re
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.generation import decode_state, prefill
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import decode as DK

ss =pytest.importorskip("scipy.stats")

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "opendiloco_b200" / "csrc"
ALPHA = 1e-4


# ------------------------------------------------------------------------------------------------ proposals
def _histories(B: int, Smax: int, seed: int):
    """B planted histories (int32 [B, Smax], lengths L [B]): lengths at and around 127 / 128 / 1024 and up to Smax, small
    alphabets (many matches), runs of distinct tokens (no match), a planted repeat of a long span, L = 1 and 2."""
    g = torch.Generator().manual_seed(seed)
    lengths = [1, 2, 3, 126, 127, 128, 129, 1023, 1024, 1025, Smax - 1, Smax]
    lengths += torch.randint(4, Smax + 1, (B - len(lengths),), generator=g).tolist()
    hist = torch.full((B, Smax), -5, dtype=torch.int32)            # junk past every history: must never be read
    for b, L in enumerate(lengths):
        kind = b % 4
        if kind == 0:
            h = torch.randint(0, 3, (L,), generator=g)
        elif kind == 1:
            h = torch.randint(0, 40, (L,), generator=g)
        elif kind == 2:
            h = torch.randperm(max(L, 1), generator=g)[:L] + 100     # distinct: no match at any n
        else:
            h = torch.randint(0, 32000, (L,), generator=g)
            if L > 40:                                             # the last 12 tokens also occur at a random earlier start
                s = int(torch.randint(0, L - 30, (1,), generator=g))
                h[L - 12:] = h[s:s + 12]
        hist[b, :L] = h.int()
    return hist, torch.tensor(lengths, dtype=torch.int32)


@pytest.mark.parametrize("K,ngram", [(1, 1), (4, 2), (7, 3), (7, 8), (3, 64)])
def test_lookup_propose_kernel_matches_reference(K, ngram):
    B, Smax = 64, 2048
    hist, lens = _histories(B, Smax, seed=K * 100 + ngram)
    pos = lens - 1
    fin = torch.zeros(B, dtype=torch.int32)
    fin[[5, 17, 40]] = 1
    eos = [1, 7]                                                   # cuts candidates in the small-alphabet rows
    ictl, _ = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, eos, "cpu")
    g = torch.Generator().manual_seed(1)
    tok0 = torch.randint(0, 32000, ((K + 1) * B,), generator=g)
    cnt0 = torch.randint(0, 8, (B,), generator=g, dtype=torch.int32)
    prop0 = torch.randint(0, 100, (B,), generator=g)
    ref = [tok0.clone(), cnt0.clone(), prop0.clone()]
    DK.lookup_propose_reference(hist, pos, fin, ictl, *ref, ngram)
    got = [tok0.cuda(), cnt0.cuda(), prop0.cuda()]
    DK.lookup_propose(hist.cuda(), pos.cuda(), fin.cuda(), ictl.cuda(), *got, ngram)
    torch.cuda.synchronize()
    for name, r, x in zip(("tok", "cnt", "proposed"), ref, got):
        assert torch.equal(x.cpu(), r), name
    c = ref[1]
    live = fin == 0
    print(f"K={K} ngram={ngram}: candidate counts of live rows {torch.bincount(c[live], minlength=K + 1).tolist()}")
    assert bool((c[live] == 0).any()) and bool((c[live] > 0).any())
    assert torch.equal(ref[0].view(K + 1, B)[:, ~live], tok0.view(K + 1, B)[:, ~live])   # finished rows left alone


# ------------------------------------------------------------------------------------------------ point-mass acceptance
def _run_accept(plog, tok, ctl, pos, gen, fin, cnt, max_new, out_w, hist):
    B = pos.shape[0]
    ictl, fctl = ctl
    st = dict(tok=tok.clone(), pos=pos.clone(), gen=gen.clone(), fin=fin.clone(), hist=hist.clone(),
              out=torch.zeros(B, out_w, dtype=torch.int64, device=pos.device),
              stats=torch.zeros(B, 2, dtype=torch.int64, device=pos.device))
    DK.accept(plog, None, ictl, fctl, st["tok"], st["pos"], st["gen"], st["fin"], st["out"], max_new, None, st["stats"], cnt=cnt,
              hist=st["hist"])
    return st


@pytest.mark.parametrize("K", [1, 4, 7])
def test_point_mass_accept_greedy_matches_reference(K):
    V, B = 32000, 64
    g = torch.Generator(device="cuda").manual_seed(K)
    plog = (3 * torch.randn((K + 1) * B, V, device="cuda", generator=g)).bfloat16()
    am = plog.float().view(K + 1, B, V).argmax(dim=-1)
    cnt = (torch.arange(B, device="cuda") % (K + 1)).int()         # every count 0..K
    tok = torch.zeros(K + 1, B, dtype=torch.int64, device="cuda")
    tok[1:] = am[:K]
    for b in range(B):
        c = int(cnt[b])
        tok[1 + c:, b] = 0                                         # fillers
        s = (b // (K + 1)) % (K + 1)                               # a wrong candidate at slot s (s >= c: none)
        if s < c:
            tok[1 + s, b] = (am[s, b] + 1) % V
    eos = int(am[0, 3])                                            # row 3 emits an EOS
    ctl = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, [eos], "cuda")
    pos = torch.randint(5, 100, (B,), dtype=torch.int32, device="cuda")
    gen = torch.randint(1, 10, (B,), dtype=torch.int32, device="cuda")
    gen[7] = 11                                                    # row 7 reaches max_new inside its block
    fin = torch.zeros(B, dtype=torch.int32, device="cuda")
    fin[9] = 1
    hist = torch.randint(0, V, (B, 128), dtype=torch.int32, device="cuda")
    got = _run_accept(plog, tok.view(-1), ctl, pos, gen, fin, cnt, 12, 16, hist)
    ref = _run_accept(plog.cpu(), tok.view(-1).cpu(), [c.cpu() for c in ctl], pos.cpu(), gen.cpu(), fin.cpu(), cnt.cpu(), 12, 16,
                      hist.cpu())
    for k in got:
        assert torch.equal(got[k].cpu(), ref[k]), k
    assert int(got["fin"][3]) == 1 and int(got["fin"][7]) == 1 and int(got["gen"][7]) == 12
    assert got["stats"][:, 1].max() <= K and bool((got["stats"][:, 1].cpu() <= cnt.cpu()).all())


def _f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


def law_probs(logits: torch.Tensor, T: float, k: int, p: float) -> torch.Tensor:
    """float64 [V]: the sampler's documented law (temperature, top-k, top-p with ties kept) on the bf16 values."""
    x = logits.double().cpu() / _f32(T)
    V = x.numel()
    w = torch.softmax(x, dim=0)
    if 0 < k < V:
        w = torch.where(x >= torch.topk(x, k).values[-1], w, 0.0)
        w = w / w.sum()
    if _f32(p) < 1.0:
        srt = torch.sort(w, descending=True).values
        m = min(int(torch.searchsorted(torch.cumsum(srt, 0), torch.tensor([_f32(p)], dtype=torch.float64))), V - 1)
        w = torch.where(w >= srt[m], w, 0.0)
        w = w / w.sum()
    return w


def chi2_binned(counts, probs, what: str) -> float:
    """Pearson chi-square of counts against probs (float64, same shape, flattened): zero counts where the law is zero;
    cells with expected count >= 5 are their own bin, the others merged in probability order into bins of >= 5."""
    o_all, p_all = np.asarray(counts, np.float64).ravel(), np.asarray(probs, np.float64).ravel()
    n = o_all.sum()
    assert o_all[p_all == 0].sum() == 0, (what, "drew an impossible outcome", np.nonzero((p_all == 0) & (o_all > 0))[0][:10])
    keep = np.nonzero(p_all > 0)[0]
    order = keep[np.argsort(-p_all[keep], kind="stable")]
    o, e = o_all[order], p_all[order] * n
    ns = int(np.argmin(e >= 5)) if not (e >= 5).all() else len(e)
    bo, be = list(o[:ns]), list(e[:ns])
    if ns < len(o):
        cum = np.cumsum(e[ns:])
        idx = np.minimum((cum // 5).astype(np.int64), max(int(cum[-1] // 5) - 1, 0))
        bo += list(np.bincount(idx, weights=o[ns:]))
        be += list(np.bincount(idx, weights=e[ns:]))
    bo, be = np.array(bo), np.array(be)
    stat = float(((bo - be) ** 2 / be).sum())
    pval = float(ss.chi2.sf(stat, len(bo) - 1))
    print(f"{what}: chi2={stat:.1f} bins={len(bo)} N={n:.0f} p={pval:.3g}")
    return pval


def _slot_logits(V: int, g: torch.Generator) -> torch.Tensor:
    """One slot's bf16 logits: 32 distinct head values 0.25 apart in (4, 12] (exact in bf16, so the top-k and top-p edges of
    WARPERS fall between distinct head values, at least 0.01 of mass from the top-p target) over a tail of about 20 % of
    the mass at temperature 1."""
    x = torch.rand(V, generator=g, dtype=torch.float64) - 2.0
    head = torch.randperm(V, generator=g)[:32]
    x[head] = 12.0 - 0.25 * torch.randperm(32, generator=g).double()
    tail = float(torch.exp(x).sum() - torch.exp(x[head]).sum())
    x[~torch.isin(torch.arange(V), head)] += float(np.log(0.25 * float(torch.exp(x[head]).sum()) / tail))
    return x.bfloat16()


WARPERS = {"none": (1.0, 0, 1.0), "combined": (0.8, 20, 0.9)}


@pytest.mark.parametrize("warp", list(WARPERS))
@pytest.mark.parametrize("c", [0, 1, 3, 4])
def test_point_mass_accept_law(c, warp):
    """The joint law of (accepted count k, emitted token t) at V = 32000 against the exact fp64 law
    P(k, t) = prod_{i<k} p_i(d_i) * p_k(t) * [t != d_k], with no exclusion at k = c (no candidate left; c = K: the bonus
    slot).  Candidates are the most likely token of their slot (probability about 0.18 without warpers, 0.29 with)."""
    V, K, rows, launches = 32000, 4, 2048, 32
    T, k, p = WARPERS[warp]
    g = torch.Generator().manual_seed(c * 10 + len(warp))
    slot = torch.stack([_slot_logits(V, g) for _ in range(K + 1)])                 # [K+1, V] bf16
    laws = [law_probs(slot[i], T, k, p) for i in range(K + 1)]
    d = [int(torch.argmax(laws[i])) for i in range(K)]
    law = torch.zeros(c + 1, V, dtype=torch.float64)
    head = 1.0
    for i in range(c + 1):
        row = laws[i].clone()
        if i < c:
            row[d[i]] = 0.0
        law[i] = head * row
        if i < c:
            head *= float(laws[i][d[i]])
    assert abs(float(law.sum()) - 1.0) < 1e-9
    plog = slot.cuda()[:, None].expand(K + 1, rows, V).contiguous().view(-1, V)
    tok = torch.zeros(K + 1, rows, dtype=torch.int64, device="cuda")
    tok[1:] = torch.tensor(d, device="cuda")[:, None]
    cnt = torch.full((rows,), c, dtype=torch.int32, device="cuda")
    z = torch.zeros(rows, dtype=torch.int32, device="cuda")
    hist = torch.zeros(rows, 16, dtype=torch.int32, device="cuda")
    counts = torch.zeros((c + 1) * V, dtype=torch.int64, device="cuda")
    for r in range(launches):
        ctl = DK.make_controls(True, T, k, p, 1000 * r + 7, 0, [], "cuda")
        st = _run_accept(plog, tok.view(-1), ctl, z, z + 1, z, cnt, 16, 16, hist)
        n_acc = st["stats"][:, 1]
        t = st["out"][torch.arange(rows, device="cuda"), 1 + n_acc]
        assert bool((st["pos"] == n_acc + 1).all()) and bool((st["hist"][torch.arange(rows, device="cuda"), 1 + n_acc] == t).all())
        counts += torch.bincount(n_acc * V + t, minlength=(c + 1) * V)
    assert chi2_binned(counts.cpu().numpy(), law.numpy(), f"point-mass accept c={c} {warp}") > ALPHA
    if c > 0:                                                      # the law of the accepted count alone
        k_counts = counts.view(c + 1, V).sum(1).cpu().numpy()
        assert ss.chisquare(k_counts, law.sum(1).numpy() * k_counts.sum()).pvalue > ALPHA


# ------------------------------------------------------------------------------------------------ generate
def _target():
    cfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=4, num_attention_heads=16, vocab_size=32000)
    return LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=1)


def _copy_prompts(B: int, P: int, seed: int) -> torch.Tensor:
    """Random prompts whose second half repeats spans of the first: the rows' histories hold n-gram matches."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, 32000, (B, P), generator=g)
    half = P // 2
    for b in range(B):
        s = int(torch.randint(0, half - 16, (1,), generator=g))
        ids[b, half:half + 16] = ids[b, s:s + 16]
        ids[b, -8:] = ids[b, s + 3:s + 11]
    return ids


def _first_gap_index(model, seq, P):
    """Per row: the first new-token index whose plain-greedy top-2 logits differ by < 0.05 (or the length)."""
    with torch.no_grad():
        logits = model(seq).logits.float()
    top2 = logits[:, P - 1:-1].topk(2, dim=-1).values
    close = (top2[..., 0] - top2[..., 1]) < 0.05
    n = seq.shape[1] - P
    return [int(torch.nonzero(close[b])[0]) if bool(close[b].any()) else n for b in range(seq.shape[0])]


def replay_bounds(prompts, new: torch.Tensor, K: int, ngram: int, eos: list[int], max_new: int):
    """Per row (rounds, accepted low, accepted high, proposed) of a greedy prompt-lookup run, from its own output and the
    rule: each emitted token is the verify pass's argmax at its slot, so every round's accepted prefix is determined,
    except in a row's last round where the accepted candidates may run past max_new (low: those inside, high: all)."""
    res = []
    for b, p in enumerate(prompts):
        R = new[b].tolist()
        h, g = list(p) + R[:1], 1
        fin = R[0] in eos or g >= max_new
        rounds = lo = hi = prop = 0
        while not fin:
            cand = DK.lookup_candidates(h, K, ngram, set(eos))
            a = 0
            while a < len(cand) and g + a < max_new and cand[a] == R[g + a]:
                a += 1
            open_end = a < len(cand) and g + a >= max_new
            rounds, lo, hi, prop = rounds + 1, lo + a, hi + (len(cand) if open_end else a), prop + len(cand)
            for x in R[g:g + a + 1]:
                if g >= max_new:
                    break
                h.append(x)
                g += 1
                if x in eos:
                    fin = True
                    break
            fin = fin or g >= max_new
        res.append((rounds, lo, hi, prop))
    return res


def _check_replay(st, prompts, new, K, ngram, eos, max_new):
    want = replay_bounds(prompts, new, K, ngram, eos, max_new)
    assert st.stats[:, 0].tolist() == [w[0] for w in want]
    assert st.proposed.tolist() == [w[3] for w in want]
    for b, w in enumerate(want):
        assert w[1] <= int(st.stats[b, 1]) <= w[2], (b, w, st.stats[b].tolist())
    assert st.verify_passes() == max(w[0] for w in want)
    return want


@pytest.mark.parametrize("graph", ["1", "0"])
def test_greedy_end_to_end(graph, monkeypatch):
    monkeypatch.setenv("ODB_CUDA_GRAPH", graph)
    target = _target()
    B, P, n_new = 4, 96, 48
    ids = _copy_prompts(B, P, 3).cuda()
    prompts = [ids[b].tolist() for b in range(B)]
    plain = target.generate(ids, max_new_tokens=n_new, eos_token_id=[])
    limit = _first_gap_index(target, plain, P)
    for Kp in (1, 4, 7):
        got = target.generate(ids, max_new_tokens=n_new, eos_token_id=[], prompt_lookup_num_tokens=Kp)
        assert torch.equal(got[:, :P], ids)
        for b in range(B):
            diff = torch.nonzero(got[b, P:] != plain[b, P:])
            if len(diff):
                assert int(diff[0]) >= limit[b], (Kp, b, int(diff[0]), limit[b])
        st = target.engine.assisted_state
        assert (st.graph is not None) == (graph == "1") and st.draft is None
        want = _check_replay(st, prompts, got[:, P:], Kp, 2, [], n_new)
        print(f"graph={graph} K={Kp}: verify passes {st.verify_passes()}, acceptance {st.acceptance_rate():.3f}, "
              f"proposed {sum(w[3] for w in want)}")
        assert sum(w[3] for w in want) > 0
    # EOS in a left-padded batch: row 0 stops at its fifth new token
    mask = torch.ones_like(ids)
    mask[1, :30] = 0
    mask[2, :90] = 0
    eos = int(plain[0, P + 4])
    ref = target.generate(ids, attention_mask=mask, max_new_tokens=n_new, eos_token_id=eos, pad_token_id=2)
    got = target.generate(ids, attention_mask=mask, max_new_tokens=n_new, eos_token_id=eos, pad_token_id=2, prompt_lookup_num_tokens=4,
                          max_matching_ngram_size=3)
    if limit[0] > 5:                                               # row 0 is not padded: plain greedy up to its first near-tie
        assert torch.equal(got[0], ref[0]) and bool((got[0, P + 5:] == 2).all())
    _check_replay(target.engine.assisted_state, [ids[b, mask[b] == 1].tolist() for b in range(B)], got[:, P:], 4, 3, [eos], n_new)
    kw = dict(max_new_tokens=n_new, do_sample=True, top_p=0.9, seed=7, eos_token_id=[], prompt_lookup_num_tokens=3)
    assert torch.equal(target.generate(ids, **kw), target.generate(ids, **kw))


SMALL = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4, vocab_size=512)
E2E_ROWS, E2E_BATCHES = 4096, 16                # 65536 sequences per configuration


def _triples(tokens: torch.Tensor) -> torch.Tensor:
    V = SMALL.vocab_size
    return (tokens[:, 0] * V + tokens[:, 1]) * V + tokens[:, 2]


def _contingency_p(a: torch.Tensor, b: torch.Tensor, what: str) -> float:
    keys, inv = torch.unique(torch.cat([a, b]), return_inverse=True)
    ca = torch.bincount(inv[: len(a)], minlength=len(keys))
    cb = torch.bincount(inv[len(a):], minlength=len(keys))
    big = (ca + cb) >= 20
    t = torch.stack([torch.cat([ca[big], ca[~big].sum()[None]]), torch.cat([cb[big], cb[~big].sum()[None]])]).cpu().numpy()
    t = t[:, t.sum(0) > 0]
    stat, pval, dof, _ = ss.chi2_contingency(t, correction=False)
    print(f"{what}: chi2={stat:.1f} dof={dof} p={pval:.3g}")
    return float(pval)


@pytest.mark.parametrize("warp", [(1.0, 0, 1.0), (1.0, 20, 0.9)])
def test_sampled_lookup_matches_plain_sampling(warp):
    """Token 1 against the fp64 law of the prefill logits; token 2 given the three most frequent t1 against the fp64 law
    of the verify pass's logits it is drawn from (slot 0 of the round after t1); without warpers, also the joint law of
    (t1, t2, t3) of lookup sampling against plain sampling (two-sample homogeneity).  The prompt is a permutation of half
    the vocabulary, so every token drawn from that half has an earlier occurrence and the row proposes the tokens after it.

    The verify pass's logits differ from the decode step's by up to one bf16 step (about 0.03 here).  With top-k and
    top-p that moves tokens across the kept-set edge, and 65536 sequences resolve the difference in the joint law for
    assisted generation just as for lookup, so with warpers each token is checked against the logits it was drawn from."""
    T, k, p = warp
    model = LlamaForCausalLM(SMALL, device="cuda", precision="bf16-mixed", seed=0)
    model.arena.p("lm_head.weight").mul_(4.0)                  # moderately peaked next-token distributions
    model.arena.sync_shadow()
    prompt = torch.randperm(SMALL.vocab_size, generator=torch.Generator().manual_seed(0))[:256]
    ids = prompt.cuda()[None].expand(E2E_ROWS, -1).contiguous()
    kw = dict(max_new_tokens=3, do_sample=True, temperature=T, top_k=k, top_p=p, eos_token_id=[])
    gen = lambda seed, **x: model.generate(ids, seed=seed, **kw, **x)[:, 256:]  # noqa: E731
    st = decode_state(model, 1, 384)                               # token 1's logits, from the same prefill program
    st.set_controls(False, 1.0, 0, 1.0, 0, 0, [])
    prefill(model, st, prompt[None].cuda(), torch.full((1,), 256, dtype=torch.int32, device="cuda"))
    law1 = law_probs(st.logits[0].clone(), T, k, p)
    plain = torch.cat([gen(100 + i) for i in range(E2E_BATCHES)])
    V = SMALL.vocab_size
    pvals = [chi2_binned(torch.bincount(plain[:, 0], minlength=V).cpu().numpy(), law1.numpy(), f"{warp} plain token 1")]
    firsts = torch.argsort(torch.bincount(plain[:, 0], minlength=V), descending=True)[:3].tolist()
    for Kp in (1, 4):
        lkw = dict(prompt_lookup_num_tokens=Kp, max_matching_ngram_size=1)
        toks = torch.cat([gen(1000 * Kp + i, **lkw) for i in range(E2E_BATCHES)])
        st = model.engine.assisted_state
        print(f"{warp} K={Kp}: acceptance {st.acceptance_rate():.3f}, proposed {int(st.proposed.sum())}")
        assert int(st.proposed.sum()) > 0 and int(st.stats[:, 1].sum()) > 0
        pvals.append(chi2_binned(torch.bincount(toks[:, 0], minlength=V).cpu().numpy(), law1.numpy(), f"{warp} lookup K={Kp} token 1"))
        # token 2 is drawn from slot 0 of the first round: its logits, from the only round of a two-token run
        last = model.generate(ids, seed=5, **dict(kw, max_new_tokens=2), **lkw)[:, 256:]
        for v in firsts:
            rows = torch.nonzero(last[:, 0] == v)[:, 0]
            assert len(rows) > 0
            law2 = law_probs(model.engine.assisted_state.plog[rows[0]].clone(), T, k, p)
            sel = toks[:, 0] == v
            pvals.append(chi2_binned(torch.bincount(toks[sel, 1], minlength=V).cpu().numpy(), law2.numpy(),
                                     f"{warp} lookup K={Kp} token 2 | t1={v}"))
        if k == 0 and p == 1.0:
            pvals.append(_contingency_p(_triples(plain), _triples(toks), f"{warp} lookup K={Kp} vs plain, joint (t1, t2, t3)"))
    assert min(pvals) > ALPHA, pvals


# ------------------------------------------------------------------------------------------------ graph and state
def _our_kernel_names() -> set[str]:
    names = set()
    for src in CSRC.glob("*.cu"):
        names |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(", src.read_text()))
    return names


_PROFILE_ROUNDS = r"""
import json, os, sys
import torch
sys.path.insert(0, os.getcwd())
from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.generation import assisted_round
from opendiloco_b200.models.llama import LlamaForCausalLM
cfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=4, num_attention_heads=16, vocab_size=32000)
target = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=1)
ids = torch.randint(3, 32000, (2, 64), device="cuda")
target.generate(ids, max_new_tokens=24, do_sample=True, top_k=40, eos_token_id=[], prompt_lookup_num_tokens=4)
st, tst = target.engine.assisted_state, target.engine.decode_state
from torch.profiler import ProfilerActivity, profile
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(3):
        assisted_round(target, None, tst, st, 24)
    torch.cuda.synchronize()
print(json.dumps({"graph": st.graph is not None, "cpu": [e.name for e in prof.events()],
                  "gpu": [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]}))
"""


def test_round_is_one_graph_of_our_kernels():
    """Three lookup rounds are three graph launches and no kernel launch, and the GPU runs only our kernels, the proposal
    kernel among them.  The profiler runs in a process of its own."""
    ours = _our_kernel_names()
    assert {"lookup_propose_kernel", "verify_attn_kernel", "accept_kernel"} <= ours
    env = dict(os.environ, ODB_CUDA_GRAPH="1")
    res = subprocess.run([sys.executable, "-c", _PROFILE_ROUNDS], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    rep = json.loads(res.stdout.strip().splitlines()[-1])
    assert rep["graph"]
    assert sum(n == "cudaGraphLaunch" for n in rep["cpu"]) == 3
    assert not [n for n in rep["cpu"] if n in ("cudaLaunchKernel", "cudaLaunchKernelExC", "cuLaunchKernel", "cuLaunchKernelEx")]
    assert rep["gpu"], "the profiler recorded no GPU activity"
    foreign = [n for n in rep["gpu"] if not any(re.search(rf"\b{k}\b", n) for k in ours)]
    assert not foreign, foreign
    for k in ("lookup_propose_kernel", "verify_attn_kernel", "accept_kernel"):
        assert any(k in n for n in rep["gpu"]), k


def test_lookup_leaves_training_state_and_releases_round_graph(monkeypatch):
    monkeypatch.setenv("ODB_CUDA_GRAPH", "1")
    cfg = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4, vocab_size=512)
    m = LlamaForCausalLM(cfg, device="cuda", seed=0)
    x = torch.randint(3, 512, (4, 128), generator=torch.Generator().manual_seed(0)).cuda()
    for _ in range(3):
        m.forward_backward(x, x, 1.0)
    key = (4, 128, 1.0, True)
    graph = m.engine._graphs[key]["graph"]
    ws = dict(m.engine._ws)
    before = [t.clone() for t in (m.arena.master, m.arena.grad, m.arena.shadow)]
    m.generate(x[:2, :50], max_new_tokens=30, do_sample=True, seed=1, prompt_lookup_num_tokens=3)
    torch.cuda.synchronize()
    assert m.engine._graphs[key]["graph"] is graph and m.engine._ws == ws
    for t0, t1 in zip(before, (m.arena.master, m.arena.grad, m.arena.shadow)):
        assert torch.equal(t0, t1)
    m.forward_backward(x, x, 1.0)
    assert m.engine._graphs[key]["graph"] is graph
    m.generate(x[:2, :50], max_new_tokens=24, eos_token_id=[], prompt_lookup_num_tokens=4)
    st = m.engine.assisted_state
    assert st.graph is not None and st.graph_target is m.engine.decode_state
    m.generate(x[:2, :50], max_new_tokens=200, eos_token_id=[])           # another Smax: a new decode state
    assert st.graph is None and st.graph_target is None
