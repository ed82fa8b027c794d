"""Prompt lookup decoding on the PyTorch reference path (CPU): the proposal rule against transformers' candidate loop,
greedy output equal to plain greedy ``generate``, the round counts replayed from the output, point-mass acceptance, seeds,
argument errors and the CLI flags."""
import os
import subprocess
import sys

import pytest
import torch

from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import decode as DK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "scripts", "generate.py")


def hf_candidates(history: list[int], K: int, max_ngram: int, eos: list[int]) -> list[int]:
    """transformers' ``PromptLookupCandidateGenerator.get_candidates`` on one row (batch 1, no max_length cut): the
    candidate tokens after the row's history."""
    input_ids = torch.tensor([history])
    input_length = input_ids.size(1)
    chosen_ids = None
    match_found = False
    for ngram_size in range(min(max_ngram, input_length - 1), 0, -1):
        windows = input_ids.unfold(dimension=1, size=ngram_size, step=1)
        ngram_tensor = input_ids[0, -ngram_size:]
        matches = (windows == ngram_tensor).all(dim=2)
        match_indices = matches.nonzero(as_tuple=True)[1]
        for idx in match_indices:
            start_idx = idx + ngram_size
            end_idx = min(start_idx + K, input_length)
            if start_idx < end_idx:
                chosen_ids = input_ids[0, start_idx:end_idx]
                match_found = True
                mask = torch.isin(chosen_ids, torch.tensor(eos, dtype=torch.long))
                match_indices_eos = torch.nonzero(mask)
                if match_indices_eos.numel() > 0:
                    chosen_ids = chosen_ids[:match_indices_eos[0].item()]
                break
        if match_found:
            break
    return [] if chosen_ids is None else chosen_ids.tolist()


def run_reference(histories: list[list[int]], K: int, ngram: int, eos: list[int], finished=None, S: int = 64):
    """lookup_propose_reference over a batch of histories; returns (tok [K+1, B], cnt, proposed)."""
    B = len(histories)
    hist = torch.full((B, S), -7, dtype=torch.int32)          # junk past every history: must never be read
    for b, h in enumerate(histories):
        hist[b, :len(h)] = torch.tensor(h, dtype=torch.int32)
    pos = torch.tensor([len(h) - 1 for h in histories], dtype=torch.int32)
    fin = torch.zeros(B, dtype=torch.int32) if finished is None else torch.tensor(finished, dtype=torch.int32)
    ictl, _ = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, eos, "cpu")
    tok = torch.full(((K + 1) * B,), 99, dtype=torch.int64)
    cnt = torch.full((B,), 5, dtype=torch.int32)
    proposed = torch.full((B,), 3, dtype=torch.int64)
    DK.lookup_propose_reference(hist, pos, fin, ictl, tok, cnt, proposed, ngram)
    return tok.view(K + 1, B), cnt, proposed


def test_planted_cases():
    K = 4
    cases = [
        ([7], []),                                        # L = 1: nothing to match
        ([1, 2, 3, 4], []),                               # no match
        ([5, 6, 9, 8, 5, 6], [9, 8, 5, 6]),               # the 2-gram at position 0
        ([1, 2, 3, 1, 2, 4, 1, 2], [3, 1, 2, 4]),         # the earliest of two matches
        ([3, 9, 4, 9], [4, 9]),                           # continuation cut short by the end of the history
        ([1, 2, 7, 3, 1, 2], [7]),                        # cut before the EOS id 3
        ([1, 2, 3, 1, 2], [3, 1, 2]),
        ([2, 2, 2, 2], [2, 2]),                           # overlapping match: s = 0 for n = 2, s + n < L
        ([1, 8, 6, 8], [6, 8]),                           # the 2-gram (6, 8) has no earlier match: n = 1 finds 8 at 1
        ([4, 3, 5, 6, 4], []),                            # the match's first follower is the EOS id: no candidates
    ]
    for h, want in cases:
        eos = [3] if h in ([1, 2, 7, 3, 1, 2], [4, 3, 5, 6, 4]) else []
        assert hf_candidates(h, K, 2, eos) == want, h
        tok, cnt, proposed = run_reference([h], K, 2, eos)
        assert int(cnt[0]) == len(want) and int(proposed[0]) == 3 + len(want)
        assert tok[1:, 0].tolist() == want + [0] * (K - len(want)), h
        assert int(tok[0, 0]) == 99                       # slot 0 is not the proposer's


@pytest.mark.parametrize("ngram", [1, 2, 3, 5])
def test_reference_matches_transformers_loop(ngram):
    g = torch.Generator().manual_seed(ngram)
    for trial in range(60):
        K = int(torch.randint(1, 8, (1,), generator=g))
        V = int(torch.randint(2, 6, (1,), generator=g))
        B = 7
        hs = [torch.randint(0, V, (int(torch.randint(1, 40, (1,), generator=g)),), generator=g).tolist() for _ in range(B)]
        eos = [] if trial % 3 == 0 else [int(torch.randint(0, V, (1,), generator=g))]
        finished = [int(b == 4) for b in range(B)]
        tok, cnt, proposed = run_reference(hs, K, ngram, eos, finished)
        for b, h in enumerate(hs):
            if finished[b]:                               # left alone
                assert tok[1:, b].tolist() == [99] * K and int(cnt[b]) == 5 and int(proposed[b]) == 3
                continue
            want = hf_candidates(h, K, ngram, eos)
            assert DK.lookup_candidates(h, K, ngram, set(eos)) == want
            assert int(cnt[b]) == len(want) and int(proposed[b]) == 3 + len(want)
            assert tok[1:, b].tolist() == want + [0] * (K - len(want)), (h, K, ngram, eos)


def _cfg(layers=2, vocab=16, max_pos=96):
    return LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=layers, num_attention_heads=2, vocab_size=vocab,
                       max_position_embeddings=max_pos)


def _ragged_batch(V, B=4, P=9, seed=0):
    ids = torch.randint(1, V, (B, P), generator=torch.Generator().manual_seed(seed))
    mask = torch.ones_like(ids)
    mask[1, :2] = 0
    mask[2, :5] = 0
    mask[3, : P - 1] = 0
    return ids.masked_fill(mask == 0, 0), mask


@pytest.fixture(scope="module")
def model():
    return LlamaForCausalLM(_cfg(), precision="32-true", seed=1)


def replay(prompts: list[list[int]], ref: torch.Tensor, K: int, ngram: int, eos: list[int], max_new: int):
    """Each row's rounds, accepted and proposed counts of a greedy prompt-lookup run, from the rule alone.  ref [B, >= max_new +
    K]: each row's greedy (argmax) continuation, long enough to decide every proposal of the last round."""
    out = []
    for b, p in enumerate(prompts):
        R = ref[b].tolist()
        assert len(R) >= max_new + K
        h, g = list(p) + R[:1], 1
        fin = R[0] in eos or g >= max_new
        rounds = acc = prop = 0
        while not fin:
            cand = DK.lookup_candidates(h, K, ngram, set(eos))
            a = 0
            while a < len(cand) and cand[a] == R[g + a]:
                a += 1
            rounds, acc, prop = rounds + 1, acc + a, prop + len(cand)
            for x in R[g:g + a + 1]:
                if g >= max_new:
                    break
                h.append(x)
                g += 1
                if x in eos:
                    fin = True
                    break
            fin = fin or g >= max_new
        out.append((rounds, acc, prop))
    return out


@pytest.mark.parametrize("K", [1, 4, 7])
def test_greedy_equals_plain_and_round_replay(model, K):
    ids, mask = _ragged_batch(16)
    P, n_new = ids.shape[1], 37
    prompts = [ids[b, mask[b] == 1].tolist() for b in range(ids.shape[0])]
    for m in (None, mask):
        plain = model.generate(ids, attention_mask=m, max_new_tokens=n_new, eos_token_id=[])
        got = model.generate(ids, attention_mask=m, max_new_tokens=n_new, eos_token_id=[], prompt_lookup_num_tokens=K)
        assert torch.equal(got, plain)
    # the rounds, accepted and proposed tokens follow from the output and the rule
    long = model.generate(ids, attention_mask=mask, max_new_tokens=n_new + K + 1, eos_token_id=[])[:, P:]
    for ngram in (1, 2, 3):
        got = model.generate(ids, attention_mask=mask, max_new_tokens=n_new, eos_token_id=[], prompt_lookup_num_tokens=K,
                             max_matching_ngram_size=ngram)
        assert torch.equal(got[:, P:], long[:, :n_new])
        st = model.engine.assisted_state
        want = replay(prompts, long, K, ngram, [], n_new)
        assert st.stats[:, 0].tolist() == [w[0] for w in want]
        assert st.stats[:, 1].tolist() == [w[1] for w in want]
        assert st.proposed.tolist() == [w[2] for w in want]
        assert st.verify_passes() == max(w[0] for w in want)
        acc, prop = sum(w[1] for w in want), sum(w[2] for w in want)
        assert acc > 0 and st.acceptance_rate() == acc / prop
        assert st.verify_passes() < n_new - 1                  # accepted proposals saved verify passes
    # EOS: row 0's sixth new token; rows stop in different rounds, the rest of a row is pad
    eos = int(plain[0, P + 5])
    plain = model.generate(ids, attention_mask=mask, max_new_tokens=n_new, eos_token_id=eos, pad_token_id=15)
    got = model.generate(ids, attention_mask=mask, max_new_tokens=n_new, eos_token_id=eos, pad_token_id=15, prompt_lookup_num_tokens=K)
    assert torch.equal(got, plain)
    assert bool((got[0, P + 6:] == 15).all())
    st = model.engine.assisted_state
    want = replay(prompts, long, K, 2, [eos], n_new)
    assert [tuple(r) for r in zip(st.stats[:, 0].tolist(), st.stats[:, 1].tolist(), st.proposed.tolist())] == want


def test_return_dict_and_golden_model(ref_model_dir):
    target = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    ids, mask = _ragged_batch(target.config.vocab_size, P=12, seed=4)
    ids[:, -4:] = ids[:, 2:6]                              # a repeated span: the prompts themselves hold matches
    plain = target.generate(ids, attention_mask=mask, max_new_tokens=21)
    for K in (2, 5):
        res = target.generate(ids, attention_mask=mask, max_new_tokens=21, prompt_lookup_num_tokens=K, return_dict_in_generate=True)
        assert torch.equal(res.sequences, plain) and res.sequences_scores is None


def test_point_mass_accept_reference():
    """Greedy with planted candidates and every count 0..K, and the sampling law of (accepted count, token)."""
    V, K, B = 10, 3, 5
    p = torch.randn(K + 1, B, V, generator=torch.Generator().manual_seed(1))
    am = p.argmax(dim=-1)
    tok = torch.zeros(K + 1, B, dtype=torch.int64)
    tok[1:] = am[:K]
    cnt = torch.tensor([0, 1, 2, 3, 3], dtype=torch.int32)
    tok[3, 4] = (am[2, 4] + 1) % V                        # row 4: d_3 wrong
    for b in range(B):
        tok[1 + int(cnt[b]):, b] = 0                      # fillers
    ictl, fctl = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, [], "cpu")
    pos, gen, fin = torch.full((B,), 5, dtype=torch.int32), torch.ones(B, dtype=torch.int32), torch.zeros(B, dtype=torch.int32)
    out = torch.zeros(B, 8, dtype=torch.int64)
    stats = torch.zeros(B, 2, dtype=torch.int64)
    hist = torch.full((B, 12), -1, dtype=torch.int32)
    DK.accept(p.view(-1, V), None, ictl, fctl, tok.view(-1), pos, gen, fin, out, 8, None, stats, cnt=cnt, hist=hist)
    assert stats[:, 1].tolist() == [0, 1, 2, 3, 2]
    for b, n_acc in enumerate(stats[:, 1].tolist()):
        emitted = am[:n_acc + 1, b].tolist()
        assert out[b, 1:2 + n_acc].tolist() == emitted
        assert hist[b, 6:7 + n_acc].tolist() == emitted and int(hist[b, 7 + n_acc]) == -1
        assert int(pos[b]) == 5 + n_acc + 1

    scipy_stats = pytest.importorskip("scipy.stats")
    V, K, rows = 6, 2, 3000
    g = torch.Generator().manual_seed(3)
    logits = 1.5 * torch.randn(K + 1, V, generator=g)
    probs = torch.softmax(logits.double(), dim=-1)
    d = probs[:K].argmax(dim=-1)                          # likely candidates: both outcomes are frequent
    for c in (0, 1, 2):
        tok = torch.zeros(K + 1, rows, dtype=torch.int64)
        tok[1:] = d[:, None]
        ictl, fctl = DK.make_controls(True, 1.0, 0, 1.0, 11 + c, 0, [], "cpu")
        z = torch.zeros(rows, dtype=torch.int32)
        out = torch.zeros(rows, 8, dtype=torch.int64)
        stats = torch.zeros(rows, 2, dtype=torch.int64)
        DK.accept(logits[:, None].expand(K + 1, rows, V).reshape(-1, V), None, ictl, fctl, tok.view(-1), z.clone(), z + 1, z.clone(),
                  out, 8, None, stats, cnt=torch.full((rows,), c, dtype=torch.int32))
        k = stats[:, 1]
        t = out[torch.arange(rows), 1 + k]
        law = torch.zeros(c + 1, V, dtype=torch.float64)
        head = 1.0
        for i in range(c + 1):
            row = probs[i].clone()
            if i < c:
                row[d[i]] = 0
            law[i] = head * row
            if i < c:
                head *= float(probs[i, d[i]])
        counts = torch.zeros(c + 1, V, dtype=torch.float64)
        counts.index_put_((k, t), torch.ones(rows, dtype=torch.float64), accumulate=True)
        assert float(counts[law == 0].sum()) == 0
        keep = law > 0
        _, pval = scipy_stats.chisquare(counts[keep].numpy(), (law[keep] * rows).numpy())
        assert pval > 1e-3, (c, pval)


def test_sampling_reproducible_and_seeded(model):
    ids, mask = _ragged_batch(16, seed=6)
    kw = dict(attention_mask=mask, max_new_tokens=15, do_sample=True, temperature=1.2, top_k=10, top_p=0.9, eos_token_id=[],
              prompt_lookup_num_tokens=3)
    a, b = model.generate(ids, seed=5, **kw), model.generate(ids, seed=5, **kw)
    assert torch.equal(a, b)
    assert not torch.equal(a, model.generate(ids, seed=6, **kw))
    assert torch.equal(a[:, :9], ids)


def test_errors(model):
    ids = torch.randint(3, 16, (2, 8))
    kw = dict(max_new_tokens=4)
    for K in (0, 8, 2.0, True):
        with pytest.raises(ValueError, match="prompt_lookup_num_tokens must be"):
            model.generate(ids, prompt_lookup_num_tokens=K, **kw)
    for n in (0, DK.MAX_NGRAM + 1, 2.0, True):
        with pytest.raises(ValueError, match="max_matching_ngram_size"):
            model.generate(ids, prompt_lookup_num_tokens=2, max_matching_ngram_size=n, **kw)
    with pytest.raises(ValueError, match="assistant_model"):
        model.generate(ids, prompt_lookup_num_tokens=2, assistant_model=model, **kw)
    with pytest.raises(ValueError, match="num_beams"):
        model.generate(ids, prompt_lookup_num_tokens=2, num_beams=2, **kw)
    for proc in (dict(repetition_penalty=1.2), dict(no_repeat_ngram_size=2), dict(min_new_tokens=2, eos_token_id=3)):
        with pytest.raises(ValueError, match="not supported yet together with prompt_lookup_num_tokens"):
            model.generate(ids, prompt_lookup_num_tokens=2, **kw, **proc)
    with pytest.raises(ValueError, match="prompt_lookup_num_tokens 7 exceeds max_position_embeddings"):   # 8 + 82 + 7 > 96
        model.generate(ids, max_new_tokens=82, prompt_lookup_num_tokens=7)
    model.generate(ids, max_new_tokens=81, prompt_lookup_num_tokens=7)


def test_cli_prompt_lookup(tmp_path):
    m_dir = tmp_path / "m"
    _cfg().save_pretrained(str(m_dir))
    args = ["--model", str(m_dir), "--prompt-ids", "5 7 5 7 9", "--prompt-ids", "3", "--max-new-tokens", "13", "--eos-token-id", "-1",
            "--init-seed", "4"]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    run = lambda *a: subprocess.run([sys.executable, SCRIPT, *args, *a], capture_output=True, text=True, env=env, cwd=ROOT)  # noqa: E731
    plain = run()
    lookup = run("--prompt-lookup-num-tokens", "3", "--max-matching-ngram-size", "3")
    assert plain.returncode == 0 and lookup.returncode == 0, (plain.stderr, lookup.stderr)
    ids = lambda r: [l for l in r.stdout.splitlines() if l.startswith("ids:")]  # noqa: E731
    assert ids(plain) == ids(lookup) and len(ids(plain)) == 2
    assert "prompt lookup:" in lookup.stdout and "verify passes" in lookup.stdout
    bad = run("--prompt-lookup-num-tokens", "9")
    assert bad.returncode != 0 and "prompt_lookup_num_tokens" in bad.stderr
