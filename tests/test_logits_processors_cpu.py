"""Logits processors (``repetition_penalty``, ``no_repeat_ngram_size``, ``min_new_tokens``) on the PyTorch reference path
(CPU): token parity with transformers' ``generate`` on the golden model for greedy and beam search, the padding rule,
the all -inf rule, argument errors and the command-line flags."""
import os
import subprocess
import sys

import pytest
import torch

from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import decode as DK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "scripts", "generate.py")
PAD = 7
N_NEW = 24


@pytest.fixture(scope="module")
def models(ref_model_dir):
    tr = pytest.importorskip("transformers")
    ours = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    hf = tr.LlamaForCausalLM.from_pretrained(ref_model_dir, attn_implementation="sdpa").float().eval()
    return ours, hf


def _prompts(V, n=3, P=10, seed=0):
    return torch.randint(3, V, (n, P), generator=torch.Generator().manual_seed(seed))


def _hf(hf, ids, n_new=N_NEW, **kw):
    with torch.no_grad():
        return hf.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=n_new, do_sample=False, pad_token_id=PAD, **kw)


def _pad_to(seq, width):
    return torch.cat([seq, torch.full((seq.shape[0], width - seq.shape[1]), PAD, dtype=seq.dtype)], dim=1)


def _greedy_case(models, eos=None, **kw):
    ours, hf = models
    ids = _prompts(ours.config.vocab_size)
    got = ours.generate(ids, max_new_tokens=N_NEW, eos_token_id=eos if eos is not None else [], pad_token_id=PAD, **kw)
    ref = _hf(hf, ids, eos_token_id=eos, **kw)
    assert torch.equal(got, _pad_to(ref, got.shape[1])), (got, ref)
    plain = ours.generate(ids, max_new_tokens=N_NEW, eos_token_id=eos if eos is not None else [], pad_token_id=PAD)
    assert not torch.equal(got, plain)                 # the processor changed the output
    return got


@pytest.mark.parametrize("penalty", [0.8, 1.3, 2.0])
def test_greedy_repetition_penalty_matches_hf(models, penalty):
    _greedy_case(models, repetition_penalty=penalty)


@pytest.mark.parametrize("n", [1, 2, 3])
def test_greedy_no_repeat_ngram_matches_hf(models, n):
    _greedy_case(models, no_repeat_ngram_size=n)


def test_greedy_all_three_match_hf(models):
    ours, _ = models
    eos = _early_token(ours)
    _greedy_case(models, eos=eos, repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=6)


def _early_token(ours):
    """A token that the unconstrained greedy run emits among its first new tokens (an EOS that really ends rows)."""
    ids = _prompts(ours.config.vocab_size)
    out = ours.generate(ids, max_new_tokens=8, eos_token_id=[])[:, ids.shape[1]:]
    return int(out[0, 1])


def test_min_new_tokens_matches_hf(models):
    ours, hf = models
    eos = _early_token(ours)
    ids = _prompts(ours.config.vocab_size)
    plain = ours.generate(ids, max_new_tokens=N_NEW, eos_token_id=eos, pad_token_id=PAD)
    assert (plain[:, ids.shape[1]:] == eos).any()      # the constraint has something to forbid
    got = _greedy_case(models, eos=eos, min_new_tokens=8)
    assert not (got[:, ids.shape[1]:ids.shape[1] + 8] == eos).any()


@pytest.mark.parametrize("R", [2, 4])
def test_beam_search_matches_hf(models, R):
    ours, hf = models
    ids = _prompts(ours.config.vocab_size)
    kw = dict(num_beams=4, num_return_sequences=R, no_repeat_ngram_size=3, repetition_penalty=1.2)
    got = ours.generate(ids, max_new_tokens=N_NEW, eos_token_id=[], pad_token_id=PAD, return_dict_in_generate=True, **kw)
    with torch.no_grad():
        ref = hf.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=N_NEW, do_sample=False, pad_token_id=PAD,
                          eos_token_id=None, output_scores=True, return_dict_in_generate=True, **kw)
    assert torch.equal(got.sequences, _pad_to(ref.sequences, got.sequences.shape[1]))
    assert torch.allclose(got.sequences_scores, ref.sequences_scores.float(), atol=1e-5, rtol=0)
    plain = ours.generate(ids, max_new_tokens=N_NEW, eos_token_id=[], pad_token_id=PAD, num_beams=4, num_return_sequences=R)
    assert not torch.equal(got.sequences, plain)


def test_beam_search_min_new_tokens_matches_hf(models):
    ours, hf = models
    eos = _early_token(ours)
    ids = _prompts(ours.config.vocab_size)
    kw = dict(num_beams=4, num_return_sequences=2, min_new_tokens=6, no_repeat_ngram_size=2)
    got = ours.generate(ids, max_new_tokens=N_NEW, eos_token_id=eos, pad_token_id=PAD, return_dict_in_generate=True, **kw)
    with torch.no_grad():
        ref = hf.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=N_NEW, do_sample=False, pad_token_id=PAD,
                          eos_token_id=eos, output_scores=True, return_dict_in_generate=True, **kw)
    assert torch.equal(got.sequences, _pad_to(ref.sequences, got.sequences.shape[1]))
    assert torch.allclose(got.sequences_scores, ref.sequences_scores.float(), atol=1e-5, rtol=0)


@pytest.mark.parametrize("num_beams", [1, 4])
def test_left_padded_rows_equal_hf_alone(models, num_beams):
    """Padding is not part of a row's history: every padded row equals HF run on that row alone, unpadded."""
    ours, hf = models
    ids = _prompts(ours.config.vocab_size, P=12)
    mask = torch.ones_like(ids)
    mask[1, :4] = 0
    mask[2, :9] = 0
    ids = ids.masked_fill(mask == 0, 0)
    kw = dict(no_repeat_ngram_size=2, repetition_penalty=1.5)
    if num_beams > 1:
        kw.update(num_beams=num_beams, num_return_sequences=2)
    R = kw.get("num_return_sequences", 1)
    got = ours.generate(ids, attention_mask=mask, max_new_tokens=N_NEW, eos_token_id=[], pad_token_id=PAD, **kw)
    for b in range(ids.shape[0]):
        real = ids[b:b + 1, int((mask[b] == 0).sum()):]
        ref = _hf(hf, real, eos_token_id=None, **kw)
        assert torch.equal(got[b * R:(b + 1) * R, ids.shape[1]:], ref[:, real.shape[1]:]), b
    plain = ours.generate(ids, attention_mask=mask, max_new_tokens=N_NEW, eos_token_id=[], pad_token_id=PAD,
                          **({"num_beams": num_beams, "num_return_sequences": 2} if num_beams > 1 else {}))
    assert not torch.equal(got, plain)


def test_ngram_1_exhausts_the_vocabulary(models):
    """no_repeat_ngram_size=1 bans every token seen: past V distinct tokens every value is -inf and the row emits 0."""
    ours, _ = models
    V = ours.config.vocab_size
    ids = torch.arange(3, 3 + 40).view(1, 40)
    n_new = V - 40 + 30
    out = ours.generate(ids, max_new_tokens=n_new, eos_token_id=[], no_repeat_ngram_size=1)[0].tolist()
    first = out[:V]
    assert sorted(first) == list(range(V))             # every token exactly once until the vocabulary is used up
    assert out[V:] == [0] * (len(out) - V)             # then all -inf: token 0


def test_reference_rules():
    """process_logits_reference against a direct transcription of the documented rules, on random histories."""
    g = torch.Generator().manual_seed(0)
    rows, V, S = 6, 40, 30
    x = torch.randn(rows, V, generator=g) * 3
    hist = torch.randint(0, 6, (rows, S), generator=g)                         # small alphabet: many n-gram matches
    lens = torch.tensor([1, 2, 5, 17, 29, 30])
    ngen = torch.tensor([0, 3, 4, 5, 6, 9])
    for p, n, m in ((1.7, 0, 0), (1.0, 1, 0), (1.0, 3, 0), (0.6, 2, 5), (1.0, 31, 0), (1.3, 4, 7)):
        got = DK.process_logits_reference(x, hist, lens, ngen, p, n, m, [5, 39])
        want = x.clone()
        for r in range(rows):
            h = hist[r, :lens[r]].tolist()
            L = len(h)
            for t in set(h):
                want[r, t] = want[r, t] * p if want[r, t] < 0 else want[r, t] / p
            if n > 0 and L + 1 >= n:
                for s in range(L - n + 1):
                    if h[s:s + n - 1] == h[L - n + 1:L]:
                        want[r, h[s + n - 1]] = float("-inf")
            if ngen[r] < m:
                want[r, [5, 39]] = float("-inf")
        assert torch.equal(got, want), (p, n, m)


def test_defaults_equal_todays_output(models):
    ours, _ = models
    ids = _prompts(ours.config.vocab_size)
    a = ours.generate(ids, max_new_tokens=12, eos_token_id=[])
    b = ours.generate(ids, max_new_tokens=12, eos_token_id=[], repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0)
    assert torch.equal(a, b)
    c = ours.generate(ids, max_new_tokens=12, eos_token_id=[], num_beams=4, return_dict_in_generate=True)
    d = ours.generate(ids, max_new_tokens=12, eos_token_id=[], num_beams=4, return_dict_in_generate=True, repetition_penalty=1.0)
    assert torch.equal(c.sequences, d.sequences) and torch.equal(c.sequences_scores, d.sequences_scores)
    e = ours.generate(ids, max_new_tokens=12, do_sample=True, seed=3, eos_token_id=[])
    f = ours.generate(ids, max_new_tokens=12, do_sample=True, seed=3, eos_token_id=[], min_new_tokens=0)
    assert torch.equal(e, f)
    ictl, fctl = DK.make_controls(True, 0.7, 5, 0.9, 1, 2, [3], "cpu")
    assert ictl.tolist()[:DK.CTL_NGRAM] == [1, 5, 1, 2, 1, 3] + [0] * 7 and fctl.tolist()[:2] == pytest.approx([0.7, 0.9])


def test_sampling_with_processors_runs_and_respects_the_ban(models):
    ours, _ = models
    ids = _prompts(ours.config.vocab_size)
    out = ours.generate(ids, max_new_tokens=40, do_sample=True, temperature=1.5, top_k=0, seed=1, eos_token_id=[],
                        no_repeat_ngram_size=2)
    for row in out.tolist():
        grams = list(zip(row, row[1:]))
        assert len(grams) == len(set(grams))


def test_errors(models):
    ours, _ = models
    ids = _prompts(ours.config.vocab_size)
    for p in (0.0, -1.0, float("inf"), float("nan"), True, "2"):
        with pytest.raises(ValueError, match="repetition_penalty"):
            ours.generate(ids, max_new_tokens=2, repetition_penalty=p)
    for n in (-1, 2.0, True, DK.MAX_NGRAM + 1):
        with pytest.raises(ValueError, match="no_repeat_ngram_size"):
            ours.generate(ids, max_new_tokens=2, no_repeat_ngram_size=n)
    for m in (-1, 1.5, False):
        with pytest.raises(ValueError, match="min_new_tokens"):
            ours.generate(ids, max_new_tokens=2, min_new_tokens=m)
    for kw in (dict(repetition_penalty=1.2), dict(no_repeat_ngram_size=3), dict(min_new_tokens=2)):
        with pytest.raises(ValueError, match="not supported yet"):
            ours.generate(ids, max_new_tokens=2, assistant_model=ours, **kw)


def test_cli_flags_on_golden_model(ref_model_dir):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    args = ["--repetition-penalty", "1.4", "--no-repeat-ngram-size", "2", "--min-new-tokens", "3"]
    res = subprocess.run([sys.executable, SCRIPT, "--model", ref_model_dir, "--prompt-ids", "1 450 37 99", "--prompt-ids", "1 7",
                          "--max-new-tokens", "10", "--num-beams", "2"] + args, capture_output=True, text=True, env=env, cwd=ROOT)
    assert res.returncode == 0, res.stderr
    rows = [[int(t) for t in line.split()[1:]] for line in res.stdout.splitlines() if line.startswith("ids:")]
    model = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    ids = torch.tensor([[1, 450, 37, 99], [0, 0, 1, 7]])
    mask = torch.tensor([[1, 1, 1, 1], [0, 0, 1, 1]])
    out = model.generate(ids, attention_mask=mask, max_new_tokens=10, num_beams=2, repetition_penalty=1.4, no_repeat_ngram_size=2,
                         min_new_tokens=3)
    assert rows[0] == out[0].tolist() and rows[1] == out[1, 2:].tolist()
    plain = model.generate(ids, attention_mask=mask, max_new_tokens=10, num_beams=2)
    assert not torch.equal(out, plain)
