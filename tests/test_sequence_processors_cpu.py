"""``sequence_bias``, ``bad_words_ids``, ``min_length`` and ``min_p`` on the PyTorch reference path (CPU): token parity with
transformers' ``generate`` on the golden model for greedy and beam search (alone and with the other processors), the
padding rule, the reference min-p warper against HF's ``MinPLogitsWarper``, argument errors and the command-line flags."""
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


def _pad_to(seq, width):
    return torch.cat([seq, torch.full((seq.shape[0], width - seq.shape[1]), PAD, dtype=seq.dtype)], dim=1)


def _plain(ours, ids, n_new=N_NEW, eos=None, **kw):
    return ours.generate(ids, max_new_tokens=n_new, eos_token_id=eos if eos is not None else [], pad_token_id=PAD, **kw)


def _compare(models, ids, eos=None, num_beams=1, R=1, changed=True, **kw):
    ours, hf = models
    beam = dict(num_beams=num_beams, num_return_sequences=R) if num_beams > 1 else {}
    got = ours.generate(ids, max_new_tokens=N_NEW, eos_token_id=eos if eos is not None else [], pad_token_id=PAD,
                        return_dict_in_generate=True, **beam, **kw)
    with torch.no_grad():
        ref = hf.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=N_NEW, do_sample=False, pad_token_id=PAD,
                          eos_token_id=eos, output_scores=True, return_dict_in_generate=True, **beam, **kw)
    assert torch.equal(got.sequences, _pad_to(ref.sequences, got.sequences.shape[1])), (got.sequences, ref.sequences)
    if num_beams > 1:
        assert torch.allclose(got.sequences_scores, ref.sequences_scores.float(), atol=1e-5, rtol=0)
    if changed:
        plain = _plain(ours, ids, eos=eos, **beam)
        assert not torch.equal(got.sequences, plain)   # the processor changed the output
    return got.sequences


def _continuation(ours, ids, n=8):
    return _plain(ours, ids, n_new=n)[:, ids.shape[1]:]


def _bias_cases(ours, ids):
    """sequence_bias settings that hit the rules: a greedy continuation's pair (its prefix is the history's tail after one
    step), a sequence longer than the history, a history equal to a sequence's prefix, two sequences on one token, a bias
    on a token the repetition penalty also touches."""
    cont = _continuation(ours, ids)
    a, b, c = int(cont[0, 0]), int(cont[0, 1]), int(cont[0, 2])
    P = ids.shape[1]
    return {
        "pair": {(a, b): -30.0, (b, c): -30.0},
        "longer_than_history": {tuple(range(3, 3 + P + 2)): 50.0, (a, b): -30.0},
        "history_is_prefix": {tuple(ids[0].tolist()) + (b,): 50.0, (a,): -30.0},
        "two_on_one_token": {(b,): 4.0, (a, b): -20.0, (int(ids[0, -1]), a, b): -15.0},
        "penalised": {(int(ids[0, -1]),): 5.0, (int(ids[1, -2]), int(ids[1, -1])): 3.0},
        "list_form": [[[a], -40.0], [[b, c], -40.0]],
    }


@pytest.mark.parametrize("case", ["pair", "longer_than_history", "history_is_prefix", "two_on_one_token", "penalised", "list_form"])
@pytest.mark.parametrize("num_beams,R", [(1, 1), (4, 1), (4, 2), (4, 4)])
def test_sequence_bias_matches_hf(models, case, num_beams, R):
    ours, _ = models
    ids = _prompts(ours.config.vocab_size)
    kw = dict(sequence_bias=_bias_cases(ours, ids)[case])
    if case == "penalised":
        kw["repetition_penalty"] = 1.3
    _compare(models, ids, num_beams=num_beams, R=R, changed=case not in ("longer_than_history", "history_is_prefix") or num_beams == 1,
             **kw)


@pytest.mark.parametrize("num_beams,R", [(1, 1), (4, 1), (4, 2), (4, 4)])
def test_bad_words_matches_hf(models, num_beams, R):
    ours, _ = models
    ids = _prompts(ours.config.vocab_size)
    cont = _continuation(ours, ids)
    bad = [[int(cont[0, 0])], [int(cont[1, 0]), int(cont[1, 1])], [int(cont[2, 1]), int(cont[2, 2]), int(cont[2, 3])]]
    out = _compare(models, ids, num_beams=num_beams, R=R, bad_words_ids=bad)
    for row in out[:, ids.shape[1]:].tolist():
        assert bad[0][0] not in row


def test_bad_word_equal_to_eos_is_dropped(models):
    ours, _ = models
    ids = _prompts(ours.config.vocab_size)
    cont = _continuation(ours, ids)
    eos = int(cont[0, 1])
    assert DK.sequence_entries(None, [[eos], [eos, 5]], [eos], ours.config.vocab_size) == [((eos, 5), float("-inf"), DK.SEQ_BAN)]
    _compare(models, ids, eos=eos, changed=False, bad_words_ids=[[eos], [int(cont[1, 0])]])


@pytest.mark.parametrize("num_beams,R", [(1, 1), (4, 2)])
def test_min_length_matches_hf(models, num_beams, R):
    ours, _ = models
    ids = _prompts(ours.config.vocab_size)
    eos = int(_continuation(ours, ids)[0, 1])
    out = _compare(models, ids, eos=eos, num_beams=num_beams, R=R, min_length=ids.shape[1] + 6)
    assert not (out[:, ids.shape[1]:ids.shape[1] + 6] == eos).any()


@pytest.mark.parametrize("num_beams,R", [(1, 1), (4, 1), (4, 2), (4, 4)])
def test_all_processors_together_match_hf(models, num_beams, R):
    ours, _ = models
    ids = _prompts(ours.config.vocab_size)
    cont = _continuation(ours, ids)
    eos = int(cont[1, 2])
    kw = dict(repetition_penalty=1.2, no_repeat_ngram_size=3, min_new_tokens=4, min_length=ids.shape[1] + 7,
              sequence_bias={(int(cont[0, 0]),): -3.0, (int(cont[0, 0]), int(cont[0, 1])): -25.0, (int(cont[2, 0]),): 2.0},
              bad_words_ids=[[int(cont[1, 0]), int(cont[1, 1])]])
    _compare(models, ids, eos=eos, num_beams=num_beams, R=R, **kw)


@pytest.mark.parametrize("num_beams", [1, 4])
def test_left_padded_rows_equal_their_unpadded_selves(models, num_beams):
    ours, _ = models
    ids = _prompts(ours.config.vocab_size, P=12)
    mask = torch.ones_like(ids)
    mask[1, :4] = 0
    mask[2, :9] = 0
    cont = _continuation(ours, ids)
    eos = int(cont[0, 3])
    kw = dict(sequence_bias={(int(ids[1, -1]), int(cont[1, 0])): -30.0, (int(cont[2, 1]),): 3.0},
              bad_words_ids=[[int(cont[0, 0]), int(cont[0, 1])]], min_length=10, num_beams=num_beams)
    got = ours.generate(ids, attention_mask=mask, max_new_tokens=N_NEW, eos_token_id=eos, pad_token_id=PAD, **kw)
    for r in range(3):
        alone = ours.generate(ids[r:r + 1, int((mask[r] == 0).sum()):], max_new_tokens=N_NEW, eos_token_id=eos, pad_token_id=PAD, **kw)
        assert torch.equal(got[r, ids.shape[1]:], alone[0, alone.shape[1] - N_NEW:])


def test_min_p_reference_matches_hf_warper():
    tr = pytest.importorskip("transformers")
    g = torch.Generator().manual_seed(0)
    for V in (50, 1000, 32000):
        x = torch.randn(6, V, generator=g) * 3
        x[0, :V // 2] = float("-inf")                  # rows already cut by an earlier warper
        x[1, 3] = x[1, 5] = x[1].max() + 1              # a tie at the top
        for min_p in (0.0, 0.01, 0.1, 0.5, 1.0):
            ours = DK.warp_logits(x, 1.0, 0, 1.0, min_p)
            ref = x if min_p == 0 else tr.generation.logits_process.MinPLogitsWarper(min_p)(None, x.clone())
            assert torch.equal(ours, ref), (V, min_p)
    x = torch.randn(4, 500, generator=g)
    chain = [tr.TemperatureLogitsWarper(0.7), tr.TopKLogitsWarper(40), tr.TopPLogitsWarper(0.9),
             tr.generation.logits_process.MinPLogitsWarper(0.05)]
    ref = x.clone()
    for w in chain:
        ref = w(None, ref)
    assert torch.equal(DK.warp_logits(x, 0.7, 40, 0.9, 0.05), ref)


def test_min_p_sampling_runs_and_greedy_ignores_it(models):
    ours, _ = models
    ids = _prompts(ours.config.vocab_size)
    assert torch.equal(_plain(ours, ids, min_p=0.3), _plain(ours, ids))
    assert torch.equal(_plain(ours, ids, num_beams=4, min_p=0.3), _plain(ours, ids, num_beams=4))
    a = _plain(ours, ids, do_sample=True, seed=3, min_p=0.2)
    assert torch.equal(a, _plain(ours, ids, do_sample=True, seed=3, min_p=0.2))
    # min_p = 1 keeps only the top token: sampling is greedy
    assert torch.equal(_plain(ours, ids, do_sample=True, seed=3, min_p=1.0, top_k=0), _plain(ours, ids))
    out = _plain(ours, ids, do_sample=True, seed=1, min_p=0.1, prompt_lookup_num_tokens=3)
    assert out.shape == (3, ids.shape[1] + N_NEW)


def test_defaults_unchanged(models):
    ours, _ = models
    ids = _prompts(ours.config.vocab_size)
    base = _plain(ours, ids, do_sample=True, seed=5)
    assert torch.equal(base, _plain(ours, ids, do_sample=True, seed=5, sequence_bias=None, bad_words_ids=None, min_length=0, min_p=None))
    assert torch.equal(base, _plain(ours, ids, do_sample=True, seed=5, min_p=0.0, sequence_bias={}, bad_words_ids=[]))


def test_errors(models):
    ours, _ = models
    V = ours.config.vocab_size
    ids = _prompts(V)
    bad = [dict(bad_words_ids=[[V]]), dict(bad_words_ids=[[-1]]), dict(bad_words_ids=[[]]), dict(bad_words_ids=[list(range(3, 3 + 65))]),
           dict(bad_words_ids=[[3]] * (DK.MAX_SEQS + 1)), dict(bad_words_ids=[list(range(3, 3 + 64))] * 300),
           dict(sequence_bias={(3,): float("nan")}), dict(sequence_bias={(3,): float("inf")}), dict(sequence_bias={(V,): 1.0}),
           dict(sequence_bias={(): 1.0}), dict(sequence_bias=[[3, 1.0]]), dict(sequence_bias=5), dict(min_length=-1),
           dict(min_length=2.5), dict(min_p=-0.1), dict(min_p=1.5), dict(min_p="x"),
           dict(bad_words_ids=[[3]], assistant_model=ours), dict(sequence_bias={(3,): 1.0}, prompt_lookup_num_tokens=2),
           dict(min_length=5, assistant_model=ours), dict(min_length=5, prompt_lookup_num_tokens=2)]
    for kw in bad:
        with pytest.raises(ValueError):
            ours.generate(ids, max_new_tokens=4, **kw)
    with pytest.raises(ValueError, match="not supported yet together with assistant_model"):
        ours.generate(ids, max_new_tokens=4, bad_words_ids=[[3]], assistant_model=ours)
    with pytest.raises(ValueError, match="not supported yet together with prompt_lookup_num_tokens"):
        ours.generate(ids, max_new_tokens=4, min_length=3, prompt_lookup_num_tokens=2)
    # -inf is a ban, and the table holds exactly its capacity
    ours.generate(ids, max_new_tokens=2, sequence_bias={(3,): float("-inf")})
    ours.generate(ids, max_new_tokens=2, bad_words_ids=[[3 + i % 50, 4] for i in range(DK.MAX_SEQS)])


def test_cli_flags(ref_model_dir):
    cmd = [sys.executable, SCRIPT, "--model", ref_model_dir, "--device", "cpu", "--precision", "32-true", "--prompt-ids", "5 6 7 8",
           "--max-new-tokens", "6", "--bad-words-ids", "12 13;99", "--sequence-bias", "12 13:-2.5;99:1.0", "--min-length", "8"]
    out = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    assert out.returncode == 0, out.stderr
    assert out.stdout.count("ids:") == 1
    cmd += ["--do-sample", "--min-p", "0.1"]
    out = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
    assert out.returncode == 0, out.stderr
