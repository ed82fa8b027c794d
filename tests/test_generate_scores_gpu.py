"""``generate(output_scores=True, output_logits=True)`` on the sm_90a kernels (H100): the sampler's score rows against the
reference processors, chi-square tests that the sampled and accepted tokens follow softmax(score row), the beam scores
and beam indices against the beam kernel's own ranking and the reference selection, graph replay, unchanged sequences
with the flags on, FP8 options, and assisted / prompt lookup decoding against plain greedy."""
import numpy as np
import pytest
import torch
from scipy import stats

from opendiloco_b200 import _lib
from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import decode as DK

pytestmark = pytest.mark.gpu
V = 32000
PAD = 0
FLAGS = dict(return_dict_in_generate=True, output_scores=True, output_logits=True)


def _cfg(shape, layers=1):
    if shape == "150m":
        return LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=layers, num_attention_heads=16, vocab_size=V)
    return LlamaConfig(hidden_size=2048, intermediate_size=5632, num_hidden_layers=layers, num_attention_heads=32, num_key_value_heads=4,
                       vocab_size=V)


@pytest.fixture(scope="module", params=["150m", "1b"])
def model(request):
    return LlamaForCausalLM(_cfg(request.param), device="cuda", precision="bf16-mixed", seed=3)


def _prompts(n=4, P=40, seed=5):
    ids = torch.randint(3, V, (n, P), generator=torch.Generator().manual_seed(seed)).cuda()
    mask = torch.ones_like(ids)
    mask[1:2, :7] = 0                                  # left padding in rows 1 and 2, when there are
    mask[2:3, :30] = 0
    return ids, mask


def _logits(rows, seed, scale=3.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(rows, V, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _sampler_state(B, do_sample, hist_len=64, **kw):
    ictl, fctl = DK.make_controls(do_sample, kw.get("temperature", 1.0), kw.get("top_k", 0), kw.get("top_p", 1.0), 11, PAD, [],
                                  "cuda", kw.get("repetition_penalty", 1.0), 0, 0, 0, kw.get("min_p", 0.0), len(kw.get("entries", [])))
    i32 = lambda: torch.zeros(B, dtype=torch.int32, device="cuda")       # noqa: E731
    pos, gen, fin = i32() + hist_len - 1, i32(), i32()
    hist = torch.randint(0, V, (B, 128), generator=torch.Generator().manual_seed(1), dtype=torch.int32).cuda()
    hist[:] = hist[:1]                                                   # every row has the same history
    table = None
    if kw.get("entries"):
        table = DK.SeqTable("cuda")
        table.set(kw["entries"])
    return dict(ictl=ictl, fctl=fctl, pos=pos, gen=gen, finished=fin, out=torch.zeros(B, 8, dtype=torch.int64, device="cuda"),
                ids_next=torch.zeros(B, dtype=torch.int64, device="cuda"), hist=hist,
                scratch=torch.zeros(B, 2 * ((V + 31) // 32), dtype=torch.int32, device="cuda"), table=table,
                seq_scratch=torch.zeros(B, V, device="cuda") if table is not None else None)


def _run_sampler(logits, st, M=2):
    B = logits.shape[0]
    sc = DK.padding_rows(torch.empty(M, B, V, device="cuda"), PAD)
    lg = DK.padding_rows(torch.empty(M, B, V, dtype=torch.bfloat16, device="cuda"), PAD)
    DK.sample(logits, st["ictl"], st["fctl"], st["pos"], st["gen"], st["finished"], st["out"], st["ids_next"], st["hist"], st["scratch"],
              st["table"], st["seq_scratch"], score_out=sc, logit_out=lg)
    return sc, lg


# ------------------------------------------------------------------------------------------------ sampler kernel
@pytest.mark.parametrize("proc", [{}, {"repetition_penalty": 1.4}, {"repetition_penalty": 0.8, "entries": [((77,), 2.0, 0), ((5, 9), -1.5, 0), ((13,), float("-inf"), 1)]}])
def test_greedy_score_rows_equal_reference_processors(proc):
    B = 6
    logits = _logits(B, 0)
    st = _sampler_state(B, False, **proc)
    hist0 = st["hist"].clone()
    pos0 = st["pos"].clone()
    sc, lg = _run_sampler(logits, st)
    c, fc = st["ictl"].tolist(), st["fctl"].tolist()
    x = logits.float()
    if DK.processors_on(c, fc):                 # on the CPU: CUDA torch divides by a scalar through its reciprocal
        x = DK.process_logits_reference(x.cpu(), hist0.cpu(), pos0.long().cpu() + 1, torch.zeros(B), fc[DK.FCTL_PENALTY], 0, 0, [],
                                        proc.get("entries", []), 0).cuda()
    assert torch.equal(sc[0], x)
    assert torch.equal(lg[0], logits)
    assert torch.equal(st["ids_next"], x.argmax(-1))
    assert torch.equal(sc[1], DK.padding_rows(torch.empty(B, V, device="cuda"), PAD))


def _pooled_chisquare(counts, p, min_expected=5.0):
    n = counts.sum()
    e = p * n
    big = e >= min_expected
    obs = np.concatenate([counts[big], [counts[~big].sum()]])
    exp = np.concatenate([e[big], [e[~big].sum()]])
    if exp[-1] < min_expected:
        obs, exp = obs[:-1], exp[:-1]
        exp = exp * obs.sum() / exp.sum()
    if len(obs) < 2:                            # a point mass: every draw must be it
        return 1.0 if obs.sum() == n else 0.0
    return stats.chisquare(obs, exp).pvalue


WARPS = [dict(temperature=0.7, top_k=40), dict(temperature=1.2, top_p=0.9), dict(min_p=0.05, temperature=0.9),
         dict(top_k=200, top_p=0.8, min_p=0.02, repetition_penalty=1.3, entries=[((77,), 4.0, 0), ((5,), 3.0, 0)])]


@pytest.mark.parametrize("warp", WARPS)
def test_sampled_tokens_follow_softmax_of_score_row(warp):
    N = 16384
    logits = _logits(1, 1, scale=1.5).expand(N, V).contiguous()
    st = _sampler_state(N, True, **warp)
    sc, _ = _run_sampler(logits, st)
    row = sc[0, 0]
    assert torch.equal(sc[0], row.expand(N, V))                          # one row, N draws
    tok = st["ids_next"]
    assert torch.isfinite(row[tok]).all()
    p = torch.softmax(row.double(), -1).cpu().numpy()
    counts = np.bincount(tok.cpu().numpy(), minlength=V).astype(np.float64)
    assert _pooled_chisquare(counts, p) > 1e-4


@pytest.mark.parametrize("mode", ["draft", "point_mass"])
@pytest.mark.parametrize("warp", WARPS[:3])
def test_accepted_tokens_follow_softmax_of_score_row(mode, warp):
    N, K = 8192, 2
    p_rows = _logits(K + 1, 2, scale=2.5)
    plog = p_rows[:, None, :].expand(K + 1, N, V).reshape((K + 1) * N, V).contiguous()
    ictl, fctl = DK.make_controls(True, warp.get("temperature", 1.0), warp.get("top_k", 0), warp.get("top_p", 1.0), 9, PAD, [],
                                  "cuda", min_p=warp.get("min_p", 0.0))
    i32 = lambda: torch.zeros(N, dtype=torch.int32, device="cuda")      # noqa: E731
    pos, gen, fin = i32() + 10, i32(), i32()
    tok = torch.zeros((K + 1) * N, dtype=torch.int64, device="cuda")
    tok[N:] = torch.randint(0, V, (K * N,), device="cuda")
    out = torch.zeros(N, 4, dtype=torch.int64, device="cuda")
    stats_ = torch.zeros(N, 2, dtype=torch.int64, device="cuda")
    sc = DK.padding_rows(torch.empty(4, N, V, device="cuda"), PAD)
    if mode == "draft":
        qlog = _logits(K, 3, scale=2.5)[:, None, :].expand(K, N, V).reshape(K * N, V).contiguous()
        DK.accept(plog, qlog, ictl, fctl, tok, pos, gen, fin, out, 4, i32(), stats_, score_out=sc)
    else:
        cnt = torch.full((N,), K, dtype=torch.int32, device="cuda")
        DK.accept(plog, None, ictl, fctl, tok, pos, gen, fin, out, 4, None, stats_, cnt=cnt, score_out=sc)
    row = sc[0, 0]
    assert torch.equal(sc[0], row.expand(N, V))
    first = out[:, 0]
    assert torch.isfinite(row[first]).all()
    p = torch.softmax(row.double(), -1).cpu().numpy()
    counts = np.bincount(first.cpu().numpy(), minlength=V).astype(np.float64)
    assert _pooled_chisquare(counts, p) > 1e-4
    # every emitted token's column holds its slot's row, and it is finite there
    n_out = gen.long()
    for b in range(0, N, 997):
        for j in range(int(n_out[b])):
            assert torch.isfinite(sc[j, b, out[b, j]])
        for j in range(int(n_out[b]), 4):
            assert torch.equal(sc[j, b], DK.padding_rows(torch.empty(V, device="cuda"), PAD))


# ------------------------------------------------------------------------------------------------ beam kernels
# sequence_bias / bad_words_ids entries: biases large enough that biased tokens are selected, 77 also in every history
# (biased and penalised), a two-token sequence and a ban
ENTRIES = [((77,), 20.0, 0), ((123,), 16.0, 0), ((77,), -0.5, 0), ((5, 9), 8.0, 0), ((13,), float("-inf"), 1)]


@pytest.mark.parametrize("nb", [4, 8])
@pytest.mark.parametrize("proc", ["off", "history", "table"])
def test_beam_scores_and_indices_kernel(nb, proc):
    B, M = 3, 6
    rows = B * nb
    K = DK.beams_to_keep(nb, 1)
    on = proc != "off"
    entries = ENTRIES if proc == "table" else []
    ictl, fctl = DK.make_controls(False, 1.0, 0, 1.0, 0, PAD, [5], "cuda", 1.3 if on else 1.0, 2 if on else 0, 0, 0, 0.0, len(entries))
    prompt = torch.randint(0, V, (B, 16), dtype=torch.int32, device="cuda")
    prompt[:, 3], prompt[:, -1] = 77, 5                  # 77 is penalised; "5 9" matches at step 0
    plens = torch.full((B,), 16, dtype=torch.int32, device="cuda")
    table = slot_i = slot_v = None
    if entries:
        table = DK.SeqTable("cuda")
        table.set(entries)
        slot_i = torch.zeros(rows, DK.MAX_SEQS, dtype=torch.int32, device="cuda")
        slot_v = torch.zeros(rows, DK.MAX_SEQS, 2, device="cuda")
    picked = []

    def state():
        i32 = lambda *s: torch.zeros(*s, dtype=torch.int32, device="cuda")          # noqa: E731
        s = dict(run_score=torch.full((rows,), DK.NEG, device="cuda"), fin_score=torch.full((rows,), DK.NEG, device="cuda"),
                 fin_flag=i32(rows), run_seq=i32(2, rows, M) + PAD, fin_seq=i32(2, rows, M) + PAD, unsat=i32(B) + 1, done=i32(B),
                 tstep=i32(B), pos=i32(rows) + 15, ids_next=torch.zeros(rows, dtype=torch.int64, device="cuda"), parent=i32(rows),
                 run_bi=i32(2, rows, M) - 1, fin_bi=i32(2, rows, M) - 1, score_out=DK.padding_rows(torch.empty(M, rows, V, device="cuda"), PAD))
        s["run_score"].view(B, nb)[:, 0] = 0
        return s

    ker, ref = state(), state()
    ns = DK.beam_splits(V)
    part_ml = torch.zeros(rows, ns, 2, device="cuda")
    cv, ci = torch.zeros(rows, ns, 2 * K, device="cuda"), torch.zeros(rows, ns, 2 * K, dtype=torch.int32, device="cuda")
    args = lambda s: (s["run_score"], s["fin_score"], s["fin_flag"], s["run_seq"], s["fin_seq"], s["unsat"], s["done"], s["tstep"],  # noqa: E731
                      s["pos"], s["ids_next"], s["parent"])
    for t in range(M):
        logits = _logits(rows, 10 + t)
        old_rs = ker["run_score"].clone()
        DK.beam_select(logits, ictl, nb, K, 1.0, 0, M, *args(ker), part_ml, cv, ci, fctl=fctl, prompt=prompt, plens=plens, table=table,
                       slot_i=slot_i, slot_v=slot_v, score_out=ker["score_out"], run_bi=ker["run_bi"], fin_bi=ker["fin_bi"])
        DK.beam_select(logits, ictl, nb, K, 1.0, 0, M, *args(ref), fctl=fctl, prompt=prompt, plens=plens, table=table,
                       score_out=ref["score_out"], run_bi=ref["run_bi"], fin_bi=ref["fin_bi"])
        picked += ker["ids_next"].tolist()
        # the selection's own value of each new running beam, bit for bit: the parent's running score + its score row entry
        par, tok = ker["parent"].long(), ker["ids_next"]
        live = ker["run_score"] > DK.NEG / 2
        want = old_rs[par] + ker["score_out"][t][par, tok]
        assert torch.equal(ker["run_score"][live], want[live]), t
        fin = torch.isfinite(ref["score_out"][t])
        assert torch.equal(torch.isfinite(ker["score_out"][t]), fin)
        assert torch.allclose(ker["score_out"][t][fin], ref["score_out"][t][fin], atol=1e-5, rtol=1e-5)
    for k in ("ids_next", "parent", "run_seq", "fin_seq", "run_bi", "fin_bi"):
        assert torch.equal(ker[k], ref[k]), k
    if entries:                                          # the biased tokens were selected, so the check above covered them
        assert 77 in picked and 123 in picked and 13 not in picked


def _ending_eos(model, ids, mask, nb):
    """EOS ids that end every returned hypothesis early: the second tokens of the nb best two-token continuations."""
    out = model.generate(ids, attention_mask=mask, max_new_tokens=2, num_beams=nb, num_return_sequences=nb, eos_token_id=[])
    return list(dict.fromkeys(out[:, -1].tolist()))[:8]


@pytest.mark.parametrize("lp", [1.0, 0.6])
def test_beam_transition_scores_when_every_hypothesis_ends_early(model, lp):
    ids, mask = _prompts(n=1)
    nb, M = 4, 24
    eos = _ending_eos(model, ids, mask, nb)
    got = model.generate(ids, attention_mask=mask, max_new_tokens=M, num_beams=nb, num_return_sequences=nb, eos_token_id=eos,
                         pad_token_id=PAD, length_penalty=lp, early_stopping=True, **FLAGS)
    n = (got.beam_indices >= 0).sum(1)
    assert int(n.max()) < M
    ts = model.compute_transition_scores(got.sequences, got.scores, got.beam_indices)
    assert ts.shape == (nb, int(n.max()))
    assert torch.allclose(ts.sum(-1), got.sequences_scores * n.float() ** lp, rtol=1e-5, atol=0)
    P = ids.shape[1]
    for r in range(nb):
        assert int(got.sequences[r, P + int(n[r]) - 1]) in eos                 # the hypothesis ends with its EOS


@pytest.mark.parametrize("kw", [dict(), dict(do_sample=True, top_k=50), dict(num_beams=4), dict(repetition_penalty=1.2)])
def test_flags_off_capture_and_launch_nothing_new(model, kw, monkeypatch):
    ids, mask = _prompts()
    M = 24
    base = dict(attention_mask=mask, max_new_tokens=M, eos_token_id=[], pad_token_id=PAD, seed=4, **kw)
    beam = kw.get("num_beams", 1) > 1
    holder = lambda: model.engine.beam_state if beam else model.engine.decode_state          # noqa: E731
    model.generate(ids, **base)
    g, key = holder().graph, holder().graph_key
    assert g is not None and (None, None) in key                            # no score / logit buffers in the key
    model.generate(ids, **base)
    assert holder().graph is g and holder().graph_key == key                  # replayed: nothing captured
    assert holder().score_buf is None and holder().logit_buf is None
    monkeypatch.setenv("ODB_CUDA_GRAPH", "0")
    counts = []
    for flags in ({}, FLAGS, {}):
        _lib.reset_launch_count()
        model.generate(ids, **base, **flags)
        counts.append(_lib.launch_count())
    assert counts[0] == counts[2]                                              # flags off launch what they did
    assert counts[1] == counts[0] + (M if beam else 0)                         # on: one beam_scores launch per selection


# ------------------------------------------------------------------------------------------------ generate()
MODES = [dict(), dict(do_sample=True, top_k=50, temperature=0.8), dict(do_sample=True, top_p=0.9, num_return_sequences=3),
         dict(num_beams=4, num_return_sequences=2, length_penalty=0.7), dict(repetition_penalty=1.3, sequence_bias={(77,): 3.0})]


@pytest.mark.parametrize("kw", MODES)
def test_flags_do_not_change_sequences_and_graph_equals_eager(model, kw, monkeypatch):
    ids, mask = _prompts()
    base = dict(attention_mask=mask, max_new_tokens=24, eos_token_id=[17, 99], pad_token_id=PAD, seed=4, **kw)
    plain = model.generate(ids, **base)
    graphed = model.generate(ids, **base, **FLAGS)
    again = model.generate(ids, **base, **FLAGS)               # same shapes: replays
    monkeypatch.setenv("ODB_CUDA_GRAPH", "0")
    eager = model.generate(ids, **base, **FLAGS)
    assert torch.equal(graphed.sequences, plain)
    for o in (again, eager):
        assert torch.equal(o.sequences, plain)
        for a, b in zip(graphed.scores + graphed.logits, o.scores + o.logits):
            assert torch.equal(a, b)
    if kw.get("num_beams", 1) > 1:
        assert torch.equal(graphed.beam_indices, eager.beam_indices)
        ts = model.compute_transition_scores(graphed.sequences, graphed.scores, graphed.beam_indices)
        n = (graphed.beam_indices >= 0).sum(1).float()
        assert torch.allclose(ts.sum(-1), graphed.sequences_scores * n ** kw["length_penalty"], rtol=1e-5, atol=0)
    else:
        P = ids.shape[1]
        new = graphed.sequences[:, P:]
        ts = model.compute_transition_scores(graphed.sequences, graphed.scores)
        assert torch.isfinite(ts).all()
        if not kw.get("do_sample"):                             # greedy: each token is the argmax of its score row
            for t in range(new.shape[1]):
                live = graphed.scores[t][:, PAD] != 0
                assert torch.equal(graphed.scores[t].argmax(-1)[live], new[live, t])


@pytest.mark.parametrize("fp8", [dict(fp8_kv_cache=True), dict(fp8_weights=True), dict(fp8_kv_cache=True, fp8_weights=True)])
def test_fp8_scores_are_the_program_that_ran(model, fp8):
    ids, mask = _prompts()
    got = model.generate(ids, attention_mask=mask, max_new_tokens=20, eos_token_id=[], pad_token_id=PAD, **fp8, **FLAGS)
    assert torch.equal(got.sequences, model.generate(ids, attention_mask=mask, max_new_tokens=20, eos_token_id=[], pad_token_id=PAD, **fp8))
    new = got.sequences[:, ids.shape[1]:]
    for t in range(20):
        assert torch.equal(got.scores[t].argmax(-1), new[:, t])
        assert torch.equal(got.scores[t], got.logits[t])        # greedy without processors: the raw logits


@pytest.mark.parametrize("mode", ["assisted", "lookup"])
def test_assisted_and_lookup_greedy_scores_equal_plain(model, mode):
    ids, mask = _prompts()
    ids = torch.cat([ids, ids[:, -6:], ids[:, -6:]], dim=1)
    mask = torch.cat([mask, torch.ones(4, 12, dtype=mask.dtype, device="cuda")], dim=1)
    kw = dict(attention_mask=mask, max_new_tokens=24, eos_token_id=[], pad_token_id=PAD, **FLAGS)
    plain = model.generate(ids, **kw)
    extra = dict(assistant_model=model, num_assistant_tokens=3) if mode == "assisted" else dict(prompt_lookup_num_tokens=3)
    got = model.generate(ids, **extra, **kw)
    P = ids.shape[1]
    for b in range(4):
        # bf16 near-ties between the one- and multi-token attention may fork a row; compare up to its first difference
        diff = (got.sequences[b, P:] != plain.sequences[b, P:]).nonzero()
        n = int(diff[0]) if len(diff) else 24
        for t in range(n):
            a, p = got.logits[t][b], plain.logits[t][b]
            assert torch.allclose(a, p, atol=0.08, rtol=0.02), (b, t, (a - p).abs().max())
            assert torch.equal(got.scores[t][b], got.logits[t][b])
        if n < 24:
            top2 = plain.logits[n][b].topk(2).values
            assert float(top2[0] - top2[1]) < 0.1
