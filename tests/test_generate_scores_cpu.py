"""``generate(output_scores=True, output_logits=True)``, ``beam_indices`` and ``compute_transition_scores`` on the PyTorch
reference path (CPU): transformers' scores, logits and beam indices on the golden model for greedy decoding, beam search
and (teacher-forced) sampling; multi-sample, assisted and prompt lookup decoding against their plain equivalents; the
padding rows of finished rows, the defaults, argument errors and ``scripts/generate.py --print-logprobs``."""
import os
import subprocess
import sys

import pytest
import torch

from opendiloco_b200.models.llama import LlamaForCausalLM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "scripts", "generate.py")
PAD = 7
N_NEW = 12
FLAGS = dict(return_dict_in_generate=True, output_scores=True, output_logits=True)


@pytest.fixture(scope="module")
def models(ref_model_dir):
    tr = pytest.importorskip("transformers")
    ours = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    hf = tr.LlamaForCausalLM.from_pretrained(ref_model_dir, attn_implementation="sdpa").float().eval()
    return ours, hf


def _prompts(V, n=3, P=9, seed=0, padded=False):
    ids = torch.randint(3, V, (n, P), generator=torch.Generator().manual_seed(seed))
    mask = torch.ones_like(ids)
    if padded:
        mask[1, :3] = 0
        mask[2, :5] = 0
    return ids.masked_fill(mask == 0, 0), mask


def _is_padding(row):
    want = torch.full_like(row, float("-inf"))
    want[PAD] = 0.0
    return torch.equal(row, want)


def _finished_before(seq, P, eos):
    """[rows, n_new] bool: the row had emitted an EOS id before column t."""
    new = seq[:, P:]
    hit = torch.isin(new, torch.tensor(eos if isinstance(eos, list) else [eos]))
    return torch.cat([torch.zeros_like(hit[:, :1]), hit[:, :-1]], dim=1).cumsum(1) > 0


def _close(a, b):
    """Equal -inf patterns, finite values to fp32 tolerance (the two models sum in different orders)."""
    assert torch.equal(torch.isneginf(a), torch.isneginf(b))
    fin = torch.isfinite(a)
    assert torch.allclose(a[fin], b[fin], atol=2e-4, rtol=1e-4), (a[fin] - b[fin]).abs().max()


def _early_eos(ours, ids, mask):
    """A token the model emits a few steps in: an EOS id that ends some rows early."""
    out = ours.generate(ids, attention_mask=mask, max_new_tokens=6, eos_token_id=[])
    return int(out[0, ids.shape[1] + 3])


# ------------------------------------------------------------------------------------------------ greedy
@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("proc", [{}, {"repetition_penalty": 1.3}, {"no_repeat_ngram_size": 2}, {"min_new_tokens": 5},
                                  {"sequence_bias": {(11,): 2.5, (5, 9): -1.0}}, {"bad_words_ids": [[13], [4, 6]]},
                                  {"min_length": 14}])
def test_greedy_scores_and_logits_match_hf(models, padded, proc):
    ours, hf = models
    ids, mask = _prompts(ours.config.vocab_size, padded=padded)
    eos = _early_eos(ours, ids, mask)
    if padded and proc:                        # HF counts the padding as history: compare the processors on full rows
        ids, mask = _prompts(ours.config.vocab_size)
    got = ours.generate(ids, attention_mask=mask, max_new_tokens=N_NEW, eos_token_id=eos, pad_token_id=PAD, **proc, **FLAGS)
    with torch.no_grad():
        ref = hf.generate(ids, attention_mask=mask, max_new_tokens=N_NEW, do_sample=False, eos_token_id=eos, pad_token_id=PAD,
                          output_scores=True, output_logits=True, return_dict_in_generate=True, **proc)
    P, n = ids.shape[1], ref.sequences.shape[1] - ids.shape[1]
    assert torch.equal(got.sequences[:, :P + n], ref.sequences)
    assert len(got.scores) == len(got.logits) == N_NEW and got.beam_indices is None
    done = _finished_before(got.sequences, P, eos)
    for t in range(N_NEW):
        live = ~done[:, t]
        assert got.scores[t].dtype == torch.float32 and got.scores[t].shape == (3, ours.config.vocab_size)
        if t < n:
            _close(got.scores[t][live], ref.scores[t][live].float())
            _close(got.logits[t][live], ref.logits[t][live].float())
        for r in (~live).nonzero()[:, 0].tolist():
            assert _is_padding(got.scores[t][r]) and _is_padding(got.logits[t][r])


def test_padding_rows_after_eos(models):
    ours, _ = models
    ids, mask = _prompts(ours.config.vocab_size)
    eos = _early_eos(ours, ids, mask)
    got = ours.generate(ids, attention_mask=mask, max_new_tokens=N_NEW, eos_token_id=eos, pad_token_id=PAD, **FLAGS)
    done = _finished_before(got.sequences, ids.shape[1], eos)
    assert done.any() and (~done).any()
    want = torch.full((ours.config.vocab_size,), float("-inf"))
    want[PAD] = 0.0
    for r, t in done.nonzero().tolist():
        assert torch.equal(got.scores[t][r], want) and torch.equal(got.logits[t][r], want)
    ts = ours.compute_transition_scores(got.sequences, got.scores)
    assert torch.equal(ts[done], torch.zeros(int(done.sum())))
    assert torch.isfinite(ts).all()


# ------------------------------------------------------------------------------------------------ beam search
@pytest.mark.parametrize("num_beams,R", [(2, 1), (2, 2), (4, 2), (4, 4), (8, 4)])
@pytest.mark.parametrize("kw", [{}, {"length_penalty": 2.0, "early_stopping": True}, {"length_penalty": 0.5, "early_stopping": "never"},
                                {"repetition_penalty": 1.5, "no_repeat_ngram_size": 2},
                                {"sequence_bias": {(11,): 1.5}, "bad_words_ids": [[13]], "min_new_tokens": 2}])
def test_beam_scores_logits_and_indices_match_hf(models, num_beams, R, kw):
    ours, hf = models
    ids, mask = _prompts(ours.config.vocab_size, padded=not kw)
    eos = _early_eos(ours, ids, mask)
    got = ours.generate(ids, attention_mask=mask, max_new_tokens=N_NEW, eos_token_id=eos, pad_token_id=PAD, num_beams=num_beams,
                        num_return_sequences=R, **kw, **FLAGS)
    with torch.no_grad():
        ref = hf.generate(ids, attention_mask=mask, max_new_tokens=N_NEW, do_sample=False, eos_token_id=eos, pad_token_id=PAD,
                          num_beams=num_beams, num_return_sequences=R, output_scores=True, output_logits=True,
                          return_dict_in_generate=True, **kw)
    P, n = ids.shape[1], ref.sequences.shape[1] - ids.shape[1]
    assert torch.equal(got.sequences[:, :P + n], ref.sequences)
    assert got.beam_indices.dtype == torch.int64 and got.beam_indices.shape == (3 * R, N_NEW)
    bi = torch.cat([ref.beam_indices, torch.full((3 * R, N_NEW - ref.beam_indices.shape[1]), -1)], dim=1)
    assert torch.equal(got.beam_indices, bi)
    rows = 3 * num_beams
    for t in range(min(len(ref.scores), N_NEW)):
        assert got.scores[t].shape == (rows, ours.config.vocab_size)
        for r in range(rows):
            if _is_padding(got.scores[t][r]):        # the prompt was done: HF keeps computing
                continue
            _close(got.scores[t][r], ref.scores[t][r].float())
            _close(got.logits[t][r], ref.logits[t][r].float())
    ts = ours.compute_transition_scores(got.sequences, got.scores, got.beam_indices)
    want = hf.compute_transition_scores(ref.sequences, ref.scores, ref.beam_indices)     # HF's method on HF's own output
    assert ts.shape == want.shape and torch.allclose(ts, want.float(), atol=2e-4, rtol=1e-4)
    _check_sequence_scores(got, kw.get("length_penalty", 1.0))


def _check_sequence_scores(got, length_penalty):
    """compute_transition_scores sums to each hypothesis's score times its length ** length_penalty."""
    ts = LlamaForCausalLM.compute_transition_scores(_Cfg, got.sequences, got.scores, got.beam_indices)
    length = (got.beam_indices >= 0).sum(1).float()
    assert torch.allclose(ts.sum(-1), got.sequences_scores * length ** length_penalty, rtol=1e-5, atol=1e-5)
    return ts


class _Cfg:                                     # compute_transition_scores reads only config.vocab_size
    class config:
        vocab_size = 512


def _ending_eos(ours, ids, nb):
    """EOS ids that end every returned hypothesis early: the second tokens of the num_beams best two-token continuations
    (a run without EOS of two new tokens; at most 8 distinct ids).  With early_stopping=True the search then ends after
    two steps."""
    out = ours.generate(ids, max_new_tokens=2, num_beams=nb, num_return_sequences=nb, eos_token_id=[])
    return list(dict.fromkeys(out[:, -1].tolist()))[:8]


@pytest.mark.parametrize("case", ["eos33", "eos43", "beams2", "beams4", "beams8"])
def test_transition_scores_when_every_hypothesis_ends_early(models, case):
    ours, hf = models
    ids, _ = _prompts(ours.config.vocab_size, n=1)
    if case.startswith("eos"):
        nb, R, eos, lp, es = 2, 1, int(case[3:]), 1.0, False
    else:
        nb = int(case[5:])
        R, lp, es = nb, 0.5, True
        eos = _ending_eos(ours, ids, nb)
    kw = dict(max_new_tokens=N_NEW, num_beams=nb, num_return_sequences=R, eos_token_id=eos, pad_token_id=PAD, length_penalty=lp,
              early_stopping=es)
    got = ours.generate(ids, **kw, **FLAGS)
    length = (got.beam_indices >= 0).sum(1)
    assert int(length.max()) < N_NEW                 # every returned hypothesis ended before max_new_tokens
    ts = _check_sequence_scores(got, lp)
    with torch.no_grad():
        ref = hf.generate(ids, do_sample=False, output_scores=True, return_dict_in_generate=True, **kw)
    want = hf.compute_transition_scores(ref.sequences, ref.scores, ref.beam_indices)
    assert ts.shape == want.shape and torch.allclose(ts, want.float(), atol=2e-4, rtol=1e-4)
    for r in range(R):                               # the scored tokens are the hypothesis' own, EOS included
        n = int(length[r])
        tok = got.sequences[r, ids.shape[1]:ids.shape[1] + n]
        rows = got.beam_indices[r, :n]
        assert torch.equal(ts[r, :n], torch.stack([got.scores[t][rows[t], tok[t]] for t in range(n)]))


# ------------------------------------------------------------------------------------------------ sampling
@pytest.mark.parametrize("warp", [dict(temperature=0.7, top_k=20), dict(temperature=1.3, top_k=0, top_p=0.8),
                                  dict(top_k=0, min_p=0.1), dict(temperature=0.9, top_k=1),
                                  dict(temperature=0.8, top_k=30, top_p=0.9, repetition_penalty=1.2)])
def test_sampled_scores_are_hf_processors_teacher_forced(models, warp):
    tr = pytest.importorskip("transformers")
    ours, hf = models
    ids, mask = _prompts(ours.config.vocab_size)
    got = ours.generate(ids, attention_mask=mask, max_new_tokens=N_NEW, do_sample=True, seed=3, eos_token_id=[], pad_token_id=PAD,
                        **warp, **FLAGS)
    procs = tr.LogitsProcessorList()
    if warp.get("repetition_penalty", 1.0) != 1.0:
        procs.append(tr.RepetitionPenaltyLogitsProcessor(warp["repetition_penalty"]))
    if warp.get("temperature", 1.0) != 1.0:
        procs.append(tr.TemperatureLogitsWarper(warp["temperature"]))
    if warp.get("top_k", 50) > 0:
        procs.append(tr.TopKLogitsWarper(warp.get("top_k", 50)))
    if warp.get("top_p", 1.0) < 1.0:
        procs.append(tr.TopPLogitsWarper(warp["top_p"]))
    if warp.get("min_p"):
        procs.append(tr.MinPLogitsWarper(warp["min_p"]))
    P = ids.shape[1]
    with torch.no_grad():
        logits = hf(got.sequences).logits.float()
    for t in range(N_NEW):
        want = procs(got.sequences[:, :P + t], logits[:, P + t - 1].clone())
        if warp.get("top_k") == 1:               # HF's top-1 keeps ties with the argmax; ours keeps the argmax alone
            assert (torch.isfinite(got.scores[t]).sum(1) == 1).all()
            fin = torch.isfinite(got.scores[t])
            assert torch.allclose(got.scores[t][fin], want[fin], atol=2e-4, rtol=1e-4)
            continue
        _close(got.scores[t], want)
        tok = got.sequences[:, P + t]
        assert torch.isfinite(got.scores[t].gather(1, tok[:, None])).all()


def test_multi_sample_outputs_equal_repeated_prompts(models):
    ours, _ = models
    ids, mask = _prompts(ours.config.vocab_size, padded=True)
    kw = dict(max_new_tokens=N_NEW, do_sample=True, top_k=10, temperature=0.8, seed=5, eos_token_id=[], pad_token_id=PAD, **FLAGS)
    got = ours.generate(ids, attention_mask=mask, num_return_sequences=2, **kw)
    rep = ours.generate(ids.repeat_interleave(2, 0), attention_mask=mask.repeat_interleave(2, 0), **kw)
    assert torch.equal(got.sequences, rep.sequences)
    for a, b in zip(got.scores + got.logits, rep.scores + rep.logits):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ assisted / prompt lookup
@pytest.mark.parametrize("mode", ["assisted", "lookup"])
def test_assisted_and_lookup_greedy_scores_equal_plain(models, mode):
    ours, _ = models
    ids, mask = _prompts(ours.config.vocab_size, padded=True)
    ids = torch.cat([ids, ids[:, -4:], ids[:, -4:]], dim=1)         # repeats for prompt lookup to find
    mask = torch.cat([mask, torch.ones(3, 8, dtype=mask.dtype)], dim=1)
    eos = _early_eos(ours, ids, mask)
    kw = dict(max_new_tokens=N_NEW, eos_token_id=eos, pad_token_id=PAD, **FLAGS)
    plain = ours.generate(ids, attention_mask=mask, **kw)
    extra = dict(assistant_model=ours, num_assistant_tokens=3) if mode == "assisted" else dict(prompt_lookup_num_tokens=3)
    got = ours.generate(ids, attention_mask=mask, **extra, **kw)
    assert torch.equal(got.sequences, plain.sequences)
    # the reference verify attention runs one einsum over all slots, the one-token step one per token: the fp32 sums can
    # differ in the last bit (measured: at most 1.8e-7), never more
    for a, b in zip(got.scores + got.logits, plain.scores + plain.logits):
        assert torch.equal(torch.isneginf(a), torch.isneginf(b))
        assert torch.allclose(a[torch.isfinite(a)], b[torch.isfinite(a)], atol=1e-6, rtol=0)


@pytest.mark.parametrize("mode", ["assisted", "lookup"])
def test_assisted_and_lookup_sampled_scores_are_warped_rows(models, mode):
    ours, hf = models
    ids, _ = _prompts(ours.config.vocab_size)
    extra = dict(assistant_model=ours, num_assistant_tokens=3) if mode == "assisted" else dict(prompt_lookup_num_tokens=3)
    got = ours.generate(ids, max_new_tokens=N_NEW, do_sample=True, top_k=8, temperature=0.7, seed=2, eos_token_id=[],
                        pad_token_id=PAD, **extra, **FLAGS)
    P = ids.shape[1]
    with torch.no_grad():
        logits = hf(got.sequences).logits.float()
    for t in range(N_NEW):
        want = logits[:, P + t - 1] / 0.7
        want = want.masked_fill(want < want.topk(8, dim=-1).values[:, -1:], float("-inf"))
        _close(got.scores[t], want)
        _close(got.logits[t], logits[:, P + t - 1])


# ------------------------------------------------------------------------------------------------ defaults and errors
def test_defaults_unchanged_and_new_fields_none(models):
    ours, _ = models
    ids, mask = _prompts(ours.config.vocab_size, padded=True)
    for kw in ({}, {"num_beams": 3}, {"do_sample": True, "seed": 1}):
        plain = ours.generate(ids, attention_mask=mask, max_new_tokens=6, **kw)
        ignored = ours.generate(ids, attention_mask=mask, max_new_tokens=6, output_scores=True, output_logits=True, **kw)
        assert isinstance(ignored, torch.Tensor) and torch.equal(plain, ignored)
        d = ours.generate(ids, attention_mask=mask, max_new_tokens=6, return_dict_in_generate=True, **kw)
        assert torch.equal(d.sequences, plain)
        assert d.scores is None and d.logits is None and d.beam_indices is None
    only = ours.generate(ids, attention_mask=mask, max_new_tokens=6, return_dict_in_generate=True, output_logits=True)
    assert only.scores is None and len(only.logits) == 6


@pytest.mark.parametrize("name", ["output_scores", "output_logits"])
@pytest.mark.parametrize("bad", [1, 0, "yes", None])
def test_bad_flag_values_raise(models, name, bad):
    ours, _ = models
    ids, _ = _prompts(ours.config.vocab_size)
    with pytest.raises(ValueError, match=name):
        ours.generate(ids, max_new_tokens=2, return_dict_in_generate=True, **{name: bad})


def test_print_logprobs_cli(ref_model_dir):
    r = subprocess.run([sys.executable, SCRIPT, "--model", ref_model_dir, "--device", "cpu", "--precision", "32-true",
                        "--prompt-ids", "5 9 11 3", "--max-new-tokens", "5", "--print-logprobs"],
                       capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr
    line = next(l for l in r.stdout.splitlines() if l.startswith("logprobs:"))
    pairs = [p.split(":") for p in line.split()[1:]]
    assert len(pairs) == 5 and all(float(lp) <= 0.0 for _, lp in pairs)
    ids = next(l for l in r.stdout.splitlines() if l.startswith("ids:")).split()[1:]
    assert [t for t, _ in pairs] == ids[-5:]


def test_print_logprobs_cli_beam_search_ending_early(models, ref_model_dir):
    ours, _ = models
    ids, _ = _prompts(ours.config.vocab_size, n=1)
    kw = dict(max_new_tokens=N_NEW, num_beams=2, num_return_sequences=1, eos_token_id=33, pad_token_id=PAD)
    got = ours.generate(ids, **kw, return_dict_in_generate=True, output_scores=True)
    want = ours.compute_transition_scores(got.sequences, got.scores, got.beam_indices, normalize_logits=True)
    r = subprocess.run([sys.executable, SCRIPT, "--model", ref_model_dir, "--device", "cpu", "--precision", "32-true",
                        "--prompt-ids", " ".join(str(t) for t in ids[0].tolist()), "--max-new-tokens", str(N_NEW), "--num-beams", "2",
                        "--num-return-sequences", "1", "--eos-token-id", "33", "--pad-token-id", str(PAD), "--print-logprobs"],
                       capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert r.returncode == 0, r.stderr
    lines = [l for l in r.stdout.splitlines() if l.startswith("logprobs:")]
    assert len(lines) == 1
    for row, line in enumerate(lines):
        n = int((got.beam_indices[row] >= 0).sum())
        assert n < N_NEW
        pairs = [p.split(":") for p in line.split()[1:]]
        assert [int(t) for t, _ in pairs] == got.sequences[row, ids.shape[1]:ids.shape[1] + n].tolist()
        assert [float(lp) for _, lp in pairs] == pytest.approx(want[row, :n].tolist(), abs=1e-4)
