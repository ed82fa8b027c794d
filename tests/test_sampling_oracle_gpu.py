"""The decode path's random half against exact fp64 laws: ``sample_kernel`` and ``accept_kernel`` (csrc/decode_sm90.cu)
at full vocabulary size, and ``generate(do_sample=True, assistant_model=...)`` against plain sampling.

The law both kernels document (``ops/decode.py::sample``) is written out in fp64 by ``expected_probs``: logits / T, keep
the top_k largest and every token tied with the k-th, then keep the smallest set of largest probabilities whose mass
reaches top_p plus every token tied with the smallest kept one.  Two deliberate departures from HF's warpers: HF's sort
keeps only some of the tied tokens at either edge, the kernels keep them all; and a rejection whose residual
max(0, p - q) has no mass emits the target's argmax (HF would draw from a zero vector).

The kernels run 1024 threads per row.  ``draw_index`` gives thread t the contiguous segment [t * per, (t + 1) * per) of
per = ceil(V / 1024) tokens and walks inside the one segment that brackets the uniform, so the families below put their
mass on segment and warp edges, index 0, V - 1 and the last partial segment (``edge_tokens``).

Statistics: every seed is fixed, so each test passes or fails the same way every run; each statistical check prints its
p-value and fails below ALPHA = 1e-4.  Pearson chi-square bins hold an expected count of at least 5, tokens ordered by
probability; a token under 1e-6 (below what an fp32 inverse CDF with 2^-32-granular uniforms resolves) only ever goes
into a merged tail bin.  A relative bias d on a token of probability pi shifts its count by about
d * sqrt(N * pi) standard deviations; at the N of each family that is what the comments next to N state.
"""
import math

import numpy as np
import pytest
import torch

from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.generation import decode_state, prefill, step
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import decode as DK

ss = pytest.importorskip("scipy.stats")

pytestmark = pytest.mark.gpu

ALPHA = 1e-4
THREADS = 1024                                 # SAMPLE_THREADS of the sampler and the acceptance kernel
VOCABS = [1000, 1025, 32000, 50264, DK.MAX_SAMPLE_VOCAB]
# 2^20 draws per sampler case: 5 standard deviations for a 5 % bias on a token of probability 1 %
SAMPLE_DRAWS = 1 << 20
SAMPLE_ROWS = 1 << 16                          # rows per launch (one expanded logits row: no memory per row)


def f32(x: float) -> float:
    """The value the kernels read: fctl holds temperature and top_p as fp32."""
    return float(torch.tensor(x, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------ the fp64 law
def expected_probs(logits: torch.Tensor, temperature: float = 1.0, top_k: int = 0, top_p: float = 1.0) -> torch.Tensor:
    """float64 [V]: the law the sampler documents, on the bf16 values the kernel reads (see the module docstring)."""
    x = logits.detach().double().cpu() / f32(temperature)
    V = x.numel()
    p = torch.softmax(x, dim=0)
    if 0 < top_k < V:
        kth = torch.topk(x, top_k).values[-1]
        p = torch.where(x >= kth, p, 0.0)
        p = p / p.sum()
    if f32(top_p) < 1.0:
        srt = torch.sort(p, descending=True).values
        m = min(int(torch.searchsorted(torch.cumsum(srt, 0), torch.tensor([f32(top_p)], dtype=torch.float64))), V - 1)
        p = torch.where(p >= srt[m], p, 0.0)
        p = p / p.sum()
    return p


def top_p_margin(logits: torch.Tensor, temperature: float, top_k: int, top_p: float) -> float:
    """How far (in probability mass) the top-p cut sits from the nearest edge of a group of tied values.  The kernel sums
    fp32 weights, so a cut within ~1e-6 of a group edge may fall either way; the families keep it >= 1e-4 away."""
    if f32(top_p) >= 1.0:
        return 1.0
    p = expected_probs(logits, temperature, top_k, 1.0)
    vals, inv = torch.unique(p[p > 0], sorted=True, return_inverse=True)
    mass = torch.zeros(vals.numel(), dtype=torch.float64).index_add_(0, inv, p[p > 0]).flip(0)
    cum = torch.cumsum(mass, 0)
    i = int(torch.searchsorted(cum, torch.tensor([f32(top_p)], dtype=torch.float64)))
    before = float(cum[i - 1]) if i > 0 else 0.0
    return min(f32(top_p) - before, float(cum[min(i, cum.numel() - 1)]) - f32(top_p))


def edge_tokens(V: int) -> list[int]:
    """Token indices where ``draw_index`` and the block reductions have edges: 0, V - 1, the first and last index of
    several threads' segments, both sides of warp boundaries (32 segments) and the last, possibly partial, segment."""
    per = -(-V // THREADS)
    last = (V - 1) // per
    cand = {0, V - 1, per - 1, per, 2 * per - 1, 31 * per - 1, 31 * per, 32 * per - 1, 32 * per, 64 * per - 1, 64 * per,
            500 * per, 501 * per - 1, (last - 1) * per, last * per - 1, last * per}
    return sorted(c for c in cand if 0 <= c < V)


# ------------------------------------------------------------------------------------------------ families of logits
def _tail_logits(V: int, g: torch.Generator, head: torch.Tensor, tail_mass: float = 0.28) -> torch.Tensor:
    """``head`` tokens at logits in [2, 4); every other token in a tail whose total mass is about ``tail_mass``."""
    hv = 2 + 2 * torch.rand(head.numel(), generator=g, dtype=torch.float64)
    n_tail = V - head.numel()
    mean_w = (math.exp(0.5) - 1) / 0.5                     # E exp(0.5 U)
    c = math.log(tail_mass / (1 - tail_mass) * float(hv.exp().sum()) / (n_tail * mean_w))
    x = c + 0.5 * torch.rand(V, generator=g, dtype=torch.float64)
    x[head] = hv
    return x.bfloat16()


def _head(V: int, g: torch.Generator, n: int = 100) -> torch.Tensor:
    """n distinct tokens: every edge token and random others."""
    edges = edge_tokens(V)
    rest = torch.tensor([i for i in torch.randperm(V, generator=g).tolist() if i not in set(edges)][: n - len(edges)])
    return torch.cat([torch.tensor(edges), rest])


def family(name: str, V: int):
    """(bf16 logits [V], temperature, top_k, top_p).  Constructions with a top-p cut are redrawn (next seed) until the
    cut is >= 1e-4 away from every edge of a tie group, so fp32 mass sums cannot move it."""
    for attempt in range(50):
        g = torch.Generator().manual_seed(1000 * VOCABS.index(V) + 17 * attempt + sum(map(ord, name)))
        edges = torch.tensor(edge_tokens(V))
        if name.startswith("tail"):
            # ~100 head tokens and a tail of ~28 % of the mass: top_k = 100 and top_p = 0.7 must never draw the tail
            x = _tail_logits(V, g, _head(V, g))
            T, k, p = {"tail_topk": (1.0, 100, 1.0), "tail_topp": (1.0, 0, 0.7), "tail_none": (1.0, 0, 1.0),
                       "tail_combined": (0.8, 130, 0.75)}[name]
        elif name == "ties_topk":
            # the k-th value (2.5) shared by every edge token, across segments and warps: all of them are kept
            x = (torch.randn(V, generator=g) * 0.5 - 1).clamp(max=2.0)
            above = torch.tensor([i for i in torch.randperm(V, generator=g).tolist() if i not in set(edges.tolist())][:40])
            x[above] = 3 + torch.rand(40, generator=g)
            x[edges] = 2.5
            T, k, p = 1.0, 43, 1.0
        elif name == "ties_topp":
            # cumulative mass 0.45 above the tie group, 0.75 after it: top_p = 0.6 crosses inside the group
            n_g, n_a = edges.numel(), 5
            above = torch.tensor([i for i in torch.randperm(V, generator=g).tolist() if i not in set(edges.tolist())][:n_a])
            mean_w = (math.exp(0.5) - 1) / 0.5
            x = math.log(0.25 / 0.3 * n_g / ((V - n_g - n_a) * mean_w)) + 0.5 * torch.rand(V, generator=g)
            x[above] = math.log(0.45 / 0.3 * n_g / (n_a * mean_w)) + 0.5 * torch.rand(n_a, generator=g)
            x[edges] = 0.0
            T, k, p = 1.0, 0, 0.6
        elif name == "temp_low":
            # T = 0.05: edge tokens at 3 - j/16 carry weights exp(-1.25 j); everything else (<= 2) is 1e-9 or underflows
            x = torch.randn(V, generator=g).clamp(max=2.0)
            x[edges] = 3.0 - torch.arange(edges.numel()) / 16
            T, k, p = 0.05, 0, 1.0
        elif name == "temp_high":
            x = 2 * torch.randn(V, generator=g)           # T = 4: close to uniform over the vocabulary
            x[edges] = 6.0
            T, k, p = 4.0, 0, 1.0
        elif name == "peaked":
            # V - 1 holds ~0.99 of the mass; the other edge tokens are rare (~1e-4 each)
            x = torch.randn(V, generator=g) - 2
            rest = float(torch.exp(x.double()).sum())
            x[edges] = math.log(1e-4 * 100 * rest)
            x[V - 1] = math.log(99 * 1.1 * rest)
            T, k, p = 1.0, 0, 1.0
        else:
            raise ValueError(name)
        x = x.bfloat16()
        if top_p_margin(x, T, k, p) >= 1e-4:
            return x, T, k, p
    raise AssertionError(f"no well-conditioned draw of family {name} at V={V}")


# ------------------------------------------------------------------------------------------------ statistics
def chi2_binned(counts, probs, what: str) -> float:
    """Pearson chi-square of counts [V] against the law probs [V] (float64): an exact zero count wherever the law is
    zero; tokens with an expected count >= 5 and probability >= 1e-6 are their own bin, the rest (in probability order)
    merged into bins of expected count >= 5.  Prints and returns the p-value."""
    counts = np.asarray(counts, dtype=np.float64)
    probs = np.asarray(probs, dtype=np.float64)
    n = counts.sum()
    removed = probs == 0
    assert counts[removed].sum() == 0, (what, "drew removed tokens", np.nonzero(removed & (counts > 0))[0][:20])
    keep = np.nonzero(~removed)[0]
    order = keep[np.argsort(-probs[keep], kind="stable")]
    o, e = counts[order], probs[order] * n
    single = (e >= 5) & (probs[order] >= 1e-6)
    n_single = int(np.argmin(single)) if not single.all() else len(single)   # probability order: singles come first
    bo, be = list(o[:n_single]), list(e[:n_single])
    if n_single < len(o):
        cum = np.cumsum(e[n_single:])
        idx = np.minimum((cum // 5).astype(np.int64), max(int(cum[-1] // 5) - 1, 0))   # the last partial bin joins its neighbour
        bo += list(np.bincount(idx, weights=o[n_single:]))
        be += list(np.bincount(idx, weights=e[n_single:]))
    bo, be = np.array(bo), np.array(be)
    if len(bo) < 2:
        print(f"{what}: one bin, chi-square not applicable (N={n:.0f})")
        return 1.0
    stat = float(((bo - be) ** 2 / be).sum())
    pval = float(ss.chi2.sf(stat, len(bo) - 1))
    print(f"{what}: chi2={stat:.1f} bins={len(bo)} N={n:.0f} p={pval:.3g}")
    return pval


def chi2_counts(obs, expected_p, what: str) -> float:
    obs = np.asarray(obs, dtype=np.float64)
    e = np.asarray(expected_p, dtype=np.float64) * obs.sum()
    ok = e > 0
    assert obs[~ok].sum() == 0, (what, obs, e)
    stat = float(((obs[ok] - e[ok]) ** 2 / e[ok]).sum())
    pval = float(ss.chi2.sf(stat, max(int(ok.sum()) - 1, 1)))
    print(f"{what}: chi2={stat:.1f} obs={obs.astype(int).tolist()} p={pval:.3g}")
    return pval


def contingency_p(table, what: str) -> float:
    t = np.asarray(table, dtype=np.float64)
    t = t[t.sum(1) > 0][:, t.sum(0) > 0]
    if min(t.shape) < 2:
        return 1.0
    stat, pval, dof, _ = ss.chi2_contingency(t, correction=False)
    print(f"{what}: chi2={stat:.1f} dof={dof} N={t.sum():.0f} p={pval:.3g}")
    return float(pval)


def coarse_bins(probs: torch.Tensor, n_bins: int = 8) -> torch.Tensor:
    """int64 [V] token -> bin: tokens in probability order cut into n_bins groups of about equal mass."""
    order = torch.argsort(probs, descending=True, stable=True)
    cum = torch.cumsum(probs[order], 0) - probs[order]
    lut = torch.empty_like(order)
    lut[order] = (cum * n_bins).long().clamp(max=n_bins - 1)
    return lut


# ------------------------------------------------------------------------------------------------ the sampler
def _sample_call(logits, ictl, fctl, gen0: int, finished=None, pad_out: int = 1):
    B = logits.shape[0]
    z = lambda: torch.zeros(B, dtype=torch.int32, device="cuda")  # noqa: E731
    gen = torch.full((B,), gen0, dtype=torch.int32, device="cuda")
    fin = z() if finished is None else finished.clone()
    out = torch.full((B, pad_out), -7, dtype=torch.int64, device="cuda")
    ids = torch.empty(B, dtype=torch.int64, device="cuda")
    DK.sample(logits, ictl, fctl, z(), gen, fin, out, ids)
    return ids, out, fin


def sample_counts(row: torch.Tensor, T: float, k: int, p: float, n: int, seed: int) -> torch.Tensor:
    """Counts [V] of n draws of the sampler from one bf16 row, expanded to SAMPLE_ROWS rows per launch (row stride 0);
    launch c uses gen = c, so every draw has its own Philox (row, offset)."""
    V = row.numel()
    ictl, fctl = DK.make_controls(True, T, k, p, seed, 0, [], "cuda")
    counts = torch.zeros(V, dtype=torch.int64, device="cuda")
    logits = row.cuda().view(1, V).expand(SAMPLE_ROWS, V)
    for c in range(n // SAMPLE_ROWS):
        ids, _, _ = _sample_call(logits, ictl, fctl, c)
        assert 0 <= int(ids.min()) and int(ids.max()) < V, "token id out of range"
        counts += torch.bincount(ids, minlength=V)
    return counts.cpu()


def test_reference_law_matches_warpers_on_tie_free_rows():
    """expected_probs keeps the same set as HF's warpers (DK.warp_logits) wherever no two logits tie."""
    g = torch.Generator().manual_seed(0)
    for V in (1000, 32000):
        x = (torch.randperm(V, generator=g).double() * (8.0 / V))     # distinct values, exact in fp32
        for T, k, p in ((1.0, 50, 1.0), (1.0, 0, 0.9), (0.7, 200, 0.5), (2.0, 0, 0.3), (0.8, 130, 0.75)):
            ours = expected_probs(x, T, k, p) > 0
            hf = torch.isfinite(DK.warp_logits(x.float()[None], f32(T), k, f32(p)))[0]
            assert torch.equal(ours, hf), (V, T, k, p, int(ours.sum()), int(hf.sum()))


def test_expanded_rows_equal_materialised_rows():
    """``sample`` passes the row stride through, so one row expanded to R rows (stride 0) draws exactly what R
    materialised copies draw: the statistical tests below rely on it."""
    V = DK.MAX_SAMPLE_VOCAB
    row, T, k, p = family("tail_combined", V)
    ictl, fctl = DK.make_controls(True, T, k, p, 99, 0, [], "cuda")
    view = row.cuda().view(1, V).expand(512, V)
    assert view.stride() == (0, 1)
    a, _, _ = _sample_call(view, ictl, fctl, 3)
    b, _, _ = _sample_call(view.contiguous(), ictl, fctl, 3)
    assert torch.equal(a, b)


FAMILIES = ["tail_topk", "tail_topp", "tail_none", "tail_combined", "ties_topk", "ties_topp", "temp_low", "temp_high", "peaked"]


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("fam", FAMILIES)
def test_sampler_law(fam, V):
    row, T, k, p = family(fam, V)
    probs = expected_probs(row, T, k, p)
    if fam in ("tail_topk", "tail_topp"):
        head = probs > 0
        assert int(head.sum()) <= 100                    # the construction: the tail is warped away
    if fam == "ties_topk":
        assert int((probs > 0).sum()) == 40 + len(edge_tokens(V))
    counts = sample_counts(row, T, k, p, SAMPLE_DRAWS, seed=V + FAMILIES.index(fam))
    pval = chi2_binned(counts, probs, f"sample {fam} V={V} T={T} top_k={k} top_p={p}")
    assert pval > ALPHA


# ------------------------------------------------------------------------------------------------ acceptance
WARPERS = {"none": (1.0, 0, 1.0), "topk": (1.0, 100, 1.0), "topp": (1.0, 0, 0.7), "combined": (0.8, 100, 0.75)}
ACCEPT_ROWS = 4096


def accept_pair(V: int, n_slots: int, seed: int, T: float, k: int, p: float):
    """(plog bf16 [n_slots + 1, V], qlog bf16 [n_slots, V]): p_j of the tail family (each slot its own head); q_j puts 60
    of its 100 head tokens on p_j's head and 40 on tokens p_j's warpers remove, so pd = 0 rejections and residual draws
    are frequent.  Redrawn until every top-p cut is well conditioned."""
    for attempt in range(50):
        g = torch.Generator().manual_seed(seed * 101 + attempt)
        P, Q = [], []
        for j in range(n_slots + 1):
            head = _head(V, g)
            P.append(_tail_logits(V, g, head))
            if j < n_slots:
                outside = torch.tensor([i for i in torch.randperm(V, generator=g)[:400].tolist() if i not in set(head.tolist())][:40])
                qhead = torch.cat([head[torch.randperm(100, generator=g)[:60]], outside])
                Q.append(_tail_logits(V, g, qhead))
        plog, qlog = torch.stack(P), torch.stack(Q)
        if all(top_p_margin(r, T, k, p) >= 1e-4 for r in torch.cat([plog, qlog])):
            return plog, qlog
    raise AssertionError("no well-conditioned accept inputs")


def accept_call(plog, qlog, drafts, ictl, fctl, g0: int):
    """One acceptance over B = drafts.shape[1] rows (plog [(K+1)*B, V] / qlog [K*B, V] slot-major, any row stride).
    Returns (accepted count [B], emitted tokens [B, K+1]: columns past the count + 1 are not written)."""
    K, B = drafts.shape
    dev = "cuda"
    tok = torch.zeros(K + 1, B, dtype=torch.int64, device=dev)
    tok[1:] = drafts
    pos = torch.zeros(B, dtype=torch.int32, device=dev)
    gen = torch.full((B,), g0, dtype=torch.int32, device=dev)
    fin = torch.zeros(B, dtype=torch.int32, device=dev)
    W = g0 + K + 2
    out = torch.full((B, W), -1, dtype=torch.int64, device=dev)
    dpos = torch.zeros_like(pos)
    stats = torch.zeros(B, 2, dtype=torch.int64, device=dev)
    DK.accept(plog, qlog, ictl, fctl, tok.view(-1), pos, gen, fin, out, W, dpos, stats)
    n_acc = stats[:, 1]
    assert bool((stats[:, 0] == 1).all()) and bool((gen == g0 + n_acc + 1).all()) and bool((n_acc <= K).all())
    return n_acc, out[:, g0:g0 + K + 1]


def accept_stats(plog_rows, qlog_rows, T, k, p, n: int, seed: int, shared: bool):
    """Run n rows of acceptance; shared: every slot reads the same p row and q row (row stride 0), else slot j reads
    plog_rows[j] / qlog_rows[j] (materialised, ACCEPT_ROWS // 4 rows per launch)."""
    K1, V = plog_rows.shape
    K = K1 - 1
    pr = [expected_probs(r, T, k, p) for r in plog_rows]
    qr = [expected_probs(r, T, k, p) for r in qlog_rows]
    g = torch.Generator().manual_seed(seed)
    ictl, fctl = DK.make_controls(True, T, k, p, seed, 0, [], "cuda")
    B = ACCEPT_ROWS if shared else ACCEPT_ROWS // 4
    if shared:
        plog = plog_rows[0].cuda().view(1, V).expand(K1 * B, V)
        qlog = qlog_rows[0].cuda().view(1, V).expand(K * B, V)
    else:
        plog = plog_rows.cuda()[:, None].expand(K1, B, V).reshape(K1 * B, V)
        qlog = qlog_rows.cuda()[:, None].expand(K, B, V).reshape(K * B, V)
    slot_counts = torch.zeros(K1, V, dtype=torch.int64, device="cuda")
    n_acc_hist = torch.zeros(K1, dtype=torch.int64, device="cuda")
    b1 = coarse_bins(pr[0]).cuda()
    b2 = coarse_bins(pr[1]).cuda()
    pair = torch.zeros(64, dtype=torch.int64, device="cuda")
    for c in range(n // B):
        drafts = torch.stack([torch.multinomial(qr[j], B, replacement=True, generator=g) for j in range(K)]).cuda()
        n_acc, emitted = accept_call(plog, qlog, drafts, ictl, fctl, 1 + c)
        emitted_n = n_acc + 1
        assert 0 <= int(emitted[:, 0].min()) and int(emitted[:, 0].max()) < V
        n_acc_hist += torch.bincount(n_acc, minlength=K1)
        for j in range(K1):
            sel = emitted_n > j
            t = emitted[sel, j]
            assert bool(((t >= 0) & (t < V)).all()), "token id out of range"
            slot_counts[j] += torch.bincount(t, minlength=V)
        both = emitted_n >= 2
        if K >= 1:
            pair += torch.bincount(b1[emitted[both, 0]] * 8 + b2[emitted[both, 1]], minlength=64)
    return pr, qr, slot_counts.cpu(), n_acc_hist.cpu(), pair.cpu().view(8, 8)


def check_accept(pr, qr, slot_counts, n_acc_hist, pair, what: str) -> None:
    K = len(qr)
    pvals = [chi2_binned(slot_counts[j], pr[j], f"{what} emitted token {j + 1}") for j in range(K + 1)]
    alpha = [float(torch.minimum(pr[i], qr[i]).sum()) for i in range(K)]
    law = []
    reach = 1.0
    for j in range(K + 1):
        law.append(reach * (1 - alpha[j]) if j < K else reach)
        reach *= alpha[j] if j < K else 1.0
    pvals.append(chi2_counts(n_acc_hist, law, f"{what} accepted count, alpha={[round(a, 3) for a in alpha]}"))
    pvals.append(contingency_p(pair, f"{what} independence of tokens 1 and 2"))
    assert min(pvals) > ALPHA, pvals


# 2^18 rows with shared rows: per slot, 4.4 standard deviations for a 5 % bias on a token of probability 3 % (rows that
# reach slot j shrink the effective N by prod alpha)
@pytest.mark.parametrize("warp", list(WARPERS))
@pytest.mark.parametrize("K", [1, 3, 7])
@pytest.mark.parametrize("V", [32000, DK.MAX_SAMPLE_VOCAB])
def test_accept_law_shared_rows(V, K, warp):
    T, k, p = WARPERS[warp]
    plog, qlog = accept_pair(V, 1, V + K, T, k, p)
    plog = plog[:1].expand(K + 1, V)
    qlog = qlog.expand(K, V)
    res = accept_stats(plog, qlog, T, k, p, 1 << 18, seed=K * 7 + len(warp), shared=True)
    check_accept(*res, f"accept shared V={V} K={K} {warp}")


# 2^16 rows, a distinct p_j and q_j per slot: catches slot-index mistakes (a bonus drawn from p_K, a residual from q_{j+1})
@pytest.mark.parametrize("warp", ["none", "combined"])
@pytest.mark.parametrize("K", [1, 3, 7])
@pytest.mark.parametrize("V", [32000, DK.MAX_SAMPLE_VOCAB])
def test_accept_law_per_slot_rows(V, K, warp):
    T, k, p = WARPERS[warp]
    plog, qlog = accept_pair(V, K, 3 * V + K, T, k, p)
    res = accept_stats(plog, qlog, T, k, p, 1 << 16, seed=K * 11 + len(warp), shared=False)
    check_accept(*res, f"accept per-slot V={V} K={K} {warp}")


# ------------------------------------------------------------------------------------------------ assisted vs plain
SMALL = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4, vocab_size=512)
LM_HEAD_SCALE = 4.0                          # raises the logits' spread: moderately peaked next-token distributions
E2E_ROWS, E2E_BATCHES = 8192, 8              # 65536 sequences per configuration
PROMPT = [5, 77, 301, 9, 444, 23, 150, 7]
E2E_WARPERS = {"off": (1.0, 0, 1.0), "on": (1.0, 20, 0.9)}


@pytest.fixture(scope="module")
def small_models():
    ms = []
    for seed in (0, 1):
        m = LlamaForCausalLM(SMALL, device="cuda", precision="bf16-mixed", seed=seed)
        m.arena.p("lm_head.weight").mul_(LM_HEAD_SCALE)
        m.arena.sync_shadow()
        ms.append(m)
    return ms


def _generate(model, T, k, p, seed, max_new=3, **kw):
    ids = torch.tensor(PROMPT, device="cuda")[None].expand(E2E_ROWS, len(PROMPT)).contiguous()
    out = model.generate(ids, max_new_tokens=max_new, do_sample=True, temperature=T, top_k=k, top_p=p, seed=seed, eos_token_id=[],
                         **kw)
    return out[:, len(PROMPT):]


def _teacher_forced_logits(model, firsts: list[int]) -> tuple[torch.Tensor, torch.Tensor]:
    """(bf16 logits after prefill [V], bf16 logits of token 2 after one ``step`` with token 1 = firsts[i], [n, V])."""
    n = len(firsts)
    st = decode_state(model, n, 128)
    st.set_controls(False, 1.0, 0, 1.0, 0, 0, [])
    ids = torch.zeros(n, 128, dtype=torch.int64, device="cuda")
    ids[:, : len(PROMPT)] = torch.tensor(PROMPT)
    prefill(model, st, ids, torch.full((n,), len(PROMPT), dtype=torch.int32, device="cuda"))
    first = st.logits[0].clone()
    st.ids.copy_(torch.tensor(firsts, device="cuda"))
    step(model, st, graph=False)
    return first, st.logits.clone()


def _triples(tokens: torch.Tensor) -> torch.Tensor:
    V = SMALL.vocab_size
    return (tokens[:, 0] * V + tokens[:, 1]) * V + tokens[:, 2]


@pytest.mark.parametrize("warp", list(E2E_WARPERS))
def test_assisted_sampling_matches_plain_sampling(small_models, warp):
    """Tokens 1 and 2 of plain and assisted sampling against the fp64 law of the target's own logits, and the joint law
    of (t1, t2, t3) of assisted sampling against plain sampling (two-sample homogeneity).  Drafts: another model (low
    acceptance: the residual draws) and the target itself (high acceptance).

    Token 2 of plain sampling follows the decode step's logits; token 2 of assisted sampling follows the verify pass's
    logits (slot 0), which round differently in bf16.  The two differ by up to one bf16 step of the logit (printed as
    ``verify-vs-step``; on an H100: 0.024 here, 0.07 with logits scaled by 12, where 65536 sequences resolved the
    shift), so each path's token 2
    is checked against the law of the logits it actually drew from.  The per-token tests see about 10 % on a token of
    probability 5 % (5.7 standard deviations); the joint test compares the two paths and so also carries the rounding
    difference, which at LM_HEAD_SCALE = 4 stays under its resolution."""
    target, other = small_models
    T, k, p = E2E_WARPERS[warp]
    plain = torch.cat([_generate(target, T, k, p, seed=100 + i) for i in range(E2E_BATCHES)])
    V = SMALL.vocab_size
    t1_counts = torch.bincount(plain[:, 0], minlength=V)
    firsts = torch.argsort(t1_counts, descending=True)[:3].tolist()
    first_logits, second_logits = _teacher_forced_logits(target, firsts)
    law1 = expected_probs(first_logits, T, k, p)
    law2 = [expected_probs(second_logits[i], T, k, p) for i in range(len(firsts))]
    assert all(top_p_margin(x.cpu(), T, k, p) > 1e-5 for x in [first_logits, *second_logits])
    pvals = []
    runs = {"plain": plain}
    for dname, draft in (("other", other), ("self", target)):
        for Kp in (1, 4):
            runs[f"{dname} K={Kp}"] = torch.cat([_generate(target, T, k, p, seed=1000 * Kp + 10 * len(dname) + i, assistant_model=draft,
                                                           num_assistant_tokens=Kp) for i in range(E2E_BATCHES)])
            print(f"{warp} {dname} K={Kp} acceptance {target.engine.assisted_state.acceptance_rate():.3f}")
    # the verify pass's logits of token 2: slot 0 of the only round of a two-token run, for each K
    verify_law = {}
    for Kp in (1, 4):
        last = _generate(target, T, k, p, seed=5, max_new=2, assistant_model=target, num_assistant_tokens=Kp)
        plog = target.engine.assisted_state.plog
        for i, v in enumerate(firsts):
            rows = torch.nonzero(last[:, 0] == v)[:, 0]
            assert len(rows) > 0
            d = (plog[rows[0]].float() - second_logits[i].float()).abs().max().item()
            print(f"K={Kp} verify-vs-step logits of token 2 after t1={v}: max |difference| = {d:.3g}")
            assert d < 0.1
            assert top_p_margin(plog[rows[0]].cpu(), T, k, p) > 1e-5
            verify_law[Kp, i] = expected_probs(plog[rows[0]], T, k, p)
    for name, toks in runs.items():
        pvals.append(chi2_binned(torch.bincount(toks[:, 0], minlength=V).cpu(), law1, f"e2e {warp} {name} token 1"))
        for i, v in enumerate(firsts):
            sel = toks[:, 0] == v
            law = law2[i] if name == "plain" else verify_law[int(name[-1]), i]
            pvals.append(chi2_binned(torch.bincount(toks[sel, 1], minlength=V).cpu(), law, f"e2e {warp} {name} token 2 | t1={v}"))
        if name != "plain":
            a, b = _triples(plain), _triples(toks)
            keys, inv = torch.unique(torch.cat([a, b]), return_inverse=True)
            ca = torch.bincount(inv[: len(a)], minlength=len(keys))
            cb = torch.bincount(inv[len(a):], minlength=len(keys))
            big = (ca + cb) >= 20
            table = torch.stack([torch.cat([ca[big], ca[~big].sum()[None]]), torch.cat([cb[big], cb[~big].sum()[None]])])
            pvals.append(contingency_p(table.cpu().numpy(), f"e2e {warp} {name} vs plain, joint (t1, t2, t3)"))
    assert min(pvals) > ALPHA, pvals


# ------------------------------------------------------------------------------------------------ deterministic edges
def _edge_rows(V: int) -> tuple[torch.Tensor, list[int]]:
    """bf16 [6, V] rows and their argmax (ties to the lowest index): argmax at V - 1; in the last segment; a 3-way tie
    across segments and warps; a tie between index 0 and V - 1; half the row -inf; all -inf but one entry."""
    per = -(-V // THREADS)
    last = (V - 1) // per
    g = torch.Generator().manual_seed(V)
    x = torch.randn(6, V, generator=g)
    x[0, V - 1] = 9
    x[1, last * per + 1] = 9
    x[2, [33 * per + 1, 32 * per - 1, 700 * per]] = 9
    x[3, [0, V - 1]] = 9
    x[4, ::2] = float("-inf")
    x[4, V - 2] = float("-inf")
    x[5, :] = float("-inf")
    x[5, 500 * per + 3] = -3
    expect = [V - 1, last * per + 1, 32 * per - 1, 0, int(x[4].argmax()), 500 * per + 3]
    return x.bfloat16(), expect


@pytest.mark.parametrize("V", [32000, DK.MAX_SAMPLE_VOCAB])
def test_greedy_edges_and_wide_rows(V):
    rows, expect = _edge_rows(V)
    assert expect == rows.float().argmax(dim=1).tolist()
    # a row stride wider than V: the padding columns hold huge values and must never be chosen or drawn
    wide = torch.full((6, V + 40), 3e38, dtype=torch.bfloat16)
    wide[:, :V] = rows
    view = wide.cuda()[:, :V]
    assert view.stride(0) == V + 40
    for do_sample, T, k in ((False, 1.0, 0), (True, 0.7, 1)):          # greedy, and top_k = 1 with do_sample
        ictl, fctl = DK.make_controls(do_sample, T, k, 1.0, 5, 0, [], "cuda")
        ids, _, _ = _sample_call(view, ictl, fctl, 0)
        assert ids.tolist() == expect, (do_sample, k)
    # sampling on the wide view stays inside [0, V)
    ictl, fctl = DK.make_controls(True, 1.0, 0, 1.0, 5, 0, [], "cuda")
    for c in range(4):
        ids, _, _ = _sample_call(view, ictl, fctl, c)
        assert int(ids.max()) < V and int(ids.min()) >= 0
    # acceptance, greedy: K = 5 slots of edge rows (bonus: row 5), every proposal the argmax (row 0) or the first wrong
    # at slot 3 (row 1); both through the wide view
    K, B = 5, 2
    plog_w = torch.full(((K + 1) * B, V + 40), 3e38, dtype=torch.bfloat16)
    plog_w[:, :V] = rows.repeat_interleave(B, dim=0)
    plog = plog_w.cuda()[:, :V]
    qlog = plog[: K * B]
    drafts = torch.tensor([expect[:K], expect[:K]], device="cuda").T.contiguous()
    drafts[3, 1] = (expect[3] + 1) % V
    for do_sample, k in ((False, 0), (True, 1)):
        ictl, fctl = DK.make_controls(do_sample, 0.9, k, 1.0, 5, 0, [], "cuda")
        n_acc, em = accept_call(plog, qlog, drafts, ictl, fctl, 1)
        assert n_acc.tolist() == [K, 3]
        assert em[0].tolist() == expect and em[1, :4].tolist() == expect[:4]


def test_warpers_off_and_finished_rows():
    V = 50264
    row, _, _, _ = family("tail_none", V)
    logits = row.cuda().view(1, V).expand(4096, V)
    draws = []
    for k, p in ((0, 1.0), (V, 1.0), (V + 7, 1.0)):      # top_k = 0, top_k >= V and top_p = 1.0 all keep everything
        ictl, fctl = DK.make_controls(True, 1.0, k, p, 21, 0, [], "cuda")
        draws.append(_sample_call(logits, ictl, fctl, 4)[0])
    assert torch.equal(draws[0], draws[1]) and torch.equal(draws[0], draws[2])
    # finished rows emit pad (sampling and greedy), write it at out[b, gen[b]], and stay finished; the others may finish on EOS
    for do_sample in (True, False):
        ictl, fctl = DK.make_controls(do_sample, 1.0, 0, 1.0, 21, 77, [int(draws[0][1])], "cuda")
        fin = torch.zeros(4096, dtype=torch.int32, device="cuda")
        fin[::3] = 1
        ids, out, fin_after = _sample_call(logits, ictl, fctl, 0, finished=fin, pad_out=2)
        assert bool((ids[::3] == 77).all()) and bool((out[::3, 0] == 77).all()) and bool((fin_after[::3] == 1).all())
        assert bool((out[:, 1] == -7).all())
        live = fin == 0
        assert torch.equal(fin_after[live].bool(), ids[live] == int(draws[0][1]))
    # acceptance leaves finished rows alone (draft_pos = pos)
    plog, qlog = accept_pair(32000, 2, 5, 1.0, 0, 1.0)
    B, K = 4, 2
    P = plog.cuda()[:, None].expand(K + 1, B, 32000).reshape(-1, 32000)
    Q = qlog.cuda()[:, None].expand(K, B, 32000).reshape(-1, 32000)
    ictl, fctl = DK.make_controls(True, 1.0, 0, 1.0, 3, 0, [], "cuda")
    tok = torch.arange((K + 1) * B, device="cuda")
    pos = torch.full((B,), 9, dtype=torch.int32, device="cuda")
    gen = torch.full((B,), 2, dtype=torch.int32, device="cuda")
    fin = torch.tensor([1, 0, 1, 0], dtype=torch.int32, device="cuda")
    out = torch.full((B, 8), -1, dtype=torch.int64, device="cuda")
    dpos = torch.zeros_like(pos)
    stats = torch.zeros(B, 2, dtype=torch.int64, device="cuda")
    DK.accept(P, Q, ictl, fctl, tok, pos, gen, fin, out, 8, dpos, stats)
    assert bool((out[::2] == -1).all()) and pos[::2].tolist() == [9, 9] and gen[::2].tolist() == [2, 2]
    assert stats[::2].sum().item() == 0 and torch.equal(dpos, pos)
