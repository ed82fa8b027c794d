"""Assisted (speculative) generation on the PyTorch reference path (CPU): greedy output equals plain greedy ``generate``,
self-drafting accepts everything, the acceptance step samples the target's distribution, and argument errors."""
import math
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


def _cfg(layers, vocab=96, max_pos=64):
    return LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=layers, num_attention_heads=2, vocab_size=vocab,
                       max_position_embeddings=max_pos)


def _ragged_batch(V, B=4, P=7, seed=0):
    ids = torch.randint(3, V, (B, P), generator=torch.Generator().manual_seed(seed))
    mask = torch.ones_like(ids)
    mask[1, :2] = 0
    mask[2, :5] = 0
    mask[3, : P - 1] = 0
    return ids.masked_fill(mask == 0, 0), mask


@pytest.fixture(scope="module")
def pair():
    return LlamaForCausalLM(_cfg(2), precision="32-true", seed=1), LlamaForCausalLM(_cfg(1), precision="32-true", seed=2)


@pytest.mark.parametrize("K", [1, 3, 4, 7])
def test_greedy_equals_plain_generate(pair, K):
    target, draft = pair
    ids, mask = _ragged_batch(96)
    n_new = 17                                           # not a multiple of K + 1 for any K here
    plain = target.generate(ids, attention_mask=mask, max_new_tokens=n_new, eos_token_id=[])
    got = target.generate(ids, attention_mask=mask, max_new_tokens=n_new, eos_token_id=[], assistant_model=draft,
                          num_assistant_tokens=K)
    assert torch.equal(got, plain)
    # EOS inside a block: row 0's fifth new token; rows stop in different rounds, the rest of a row is pad
    eos = int(plain[0, 7 + 4])
    plain = target.generate(ids, attention_mask=mask, max_new_tokens=n_new, eos_token_id=eos, pad_token_id=95)
    got = target.generate(ids, attention_mask=mask, max_new_tokens=n_new, eos_token_id=eos, pad_token_id=95, assistant_model=draft,
                          num_assistant_tokens=K)
    assert torch.equal(got, plain)
    assert bool((got[0, 7 + 5:] == 95).all())


def test_greedy_on_golden_model(ref_model_dir):
    target = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    tcfg = target.config
    dcfg = LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=1, num_attention_heads=2,
                       vocab_size=tcfg.vocab_size, max_position_embeddings=tcfg.max_position_embeddings)
    draft = LlamaForCausalLM(dcfg, precision="32-true", seed=3)
    ids, mask = _ragged_batch(tcfg.vocab_size, P=9, seed=4)
    plain = target.generate(ids, attention_mask=mask, max_new_tokens=21)
    for K in (2, 5):
        assert torch.equal(target.generate(ids, attention_mask=mask, max_new_tokens=21, assistant_model=draft, num_assistant_tokens=K),
                           plain)


@pytest.mark.parametrize("K,n_new", [(1, 12), (3, 13), (4, 20), (7, 9)])
def test_self_draft_accepts_everything(pair, K, n_new):
    target, _ = pair
    twin = LlamaForCausalLM(_cfg(2), precision="32-true", seed=1)
    ids, mask = _ragged_batch(96, seed=5)
    plain = target.generate(ids, attention_mask=mask, max_new_tokens=n_new, eos_token_id=[])
    for draft in (target, twin):                          # the model itself, or a copy of it
        got = target.generate(ids, attention_mask=mask, max_new_tokens=n_new, eos_token_id=[], assistant_model=draft,
                              num_assistant_tokens=K)
        assert torch.equal(got, plain)
        st = target.engine.assisted_state
        assert st.acceptance_rate() == 1.0
        assert st.verify_passes() == math.ceil((n_new - 1) / (K + 1))


def test_sampling_reproducible_and_seeded(pair):
    target, draft = pair
    ids, mask = _ragged_batch(96, seed=6)
    kw = dict(attention_mask=mask, max_new_tokens=15, do_sample=True, temperature=1.2, top_k=20, top_p=0.9, eos_token_id=[],
              assistant_model=draft, num_assistant_tokens=3)
    a, b = target.generate(ids, seed=5, **kw), target.generate(ids, seed=5, **kw)
    assert torch.equal(a, b)
    assert not torch.equal(a, target.generate(ids, seed=6, **kw))
    assert torch.equal(a[:, :7], ids)


def _accept_first_tokens(p_logits, q_logits, rows, warp, seed):
    """Run the reference acceptance step on `rows` rows sharing p (slots [K+1, V]) and q ([K, V]), with proposals drawn from
    the warped q; return the first emitted token of every row."""
    K, V = q_logits.shape
    temperature, top_k, top_p = warp
    qw = torch.softmax(DK.warp_logits(q_logits, temperature, top_k, top_p), dim=-1)
    g = torch.Generator().manual_seed(seed)
    drafts = torch.stack([torch.multinomial(qw[i], rows, replacement=True, generator=g) for i in range(K)])      # [K, rows]
    tok = torch.zeros(K + 1, rows, dtype=torch.int64)
    tok[1:] = drafts
    ictl, fctl = DK.make_controls(True, temperature, top_k, top_p, seed, 0, [], "cpu")
    z = lambda: torch.zeros(rows, dtype=torch.int32)  # noqa: E731
    pos, gen, fin, dpos = z(), z() + 1, z(), z()
    out = torch.zeros(rows, 16, dtype=torch.int64)
    stats = torch.zeros(rows, 2, dtype=torch.int64)
    plog = p_logits[:, None, :].expand(K + 1, rows, V).reshape(-1, V)
    qlog = q_logits[:, None, :].expand(K, rows, V).reshape(-1, V)
    DK.accept(plog, qlog, ictl, fctl, tok.view(-1), pos, gen, fin, out, 16, dpos, stats)
    n_acc = stats[:, 1]
    assert bool((gen == 1 + n_acc + 1).all()) and bool((pos == n_acc + 1).all()) and torch.equal(dpos, pos)
    return out[:, 1]


@pytest.mark.parametrize("warp", [(1.0, 0, 1.0), (0.8, 6, 1.0), (1.3, 0, 0.7), (0.9, 8, 0.8)])
def test_acceptance_reference_samples_target_distribution(warp):
    scipy_stats = pytest.importorskip("scipy.stats")
    V, K, rows = 12, 2, 6000
    g = torch.Generator().manual_seed(7)
    p_logits = 2 * torch.randn(K + 1, V, generator=g)
    # the draft favours tokens the target's top-k / top-p removes
    q_logits = -p_logits[:K] + 0.5 * torch.randn(K, V, generator=g)
    first = _accept_first_tokens(p_logits, q_logits, rows, warp, seed=11)
    p1 = torch.softmax(DK.warp_logits(p_logits[:1].double(), *warp), dim=-1)[0]
    counts = torch.bincount(first, minlength=V).double()
    assert float(counts[p1 == 0].sum()) == 0          # no token the target's warpers removed
    keep = p1 > 0
    stat, pval = scipy_stats.chisquare(counts[keep].numpy(), (p1[keep] * rows).numpy())
    print("chi-square", warp, stat, pval)
    assert pval > 1e-3


def test_greedy_acceptance_reference():
    V, K, B = 10, 3, 4
    p = torch.randn(K + 1, B, V, generator=torch.Generator().manual_seed(1))
    am = p.argmax(dim=-1)                                 # [K+1, B]
    tok = torch.zeros(K + 1, B, dtype=torch.int64)
    tok[1:] = am[:K]
    tok[2, 1] = (am[1, 1] + 1) % V                        # row 1: d_2 wrong -> accept 1, emit the argmax of slot 1
    tok[1, 2] = (am[0, 2] + 1) % V                        # row 2: d_1 wrong -> accept 0
    ictl, fctl = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, [], "cpu")
    z = lambda: torch.zeros(B, dtype=torch.int32)  # noqa: E731
    pos, gen, fin, dpos = z() + 5, z() + 1, z(), z()
    fin[3] = 1
    out = torch.zeros(B, 8, dtype=torch.int64)
    stats = torch.zeros(B, 2, dtype=torch.int64)
    DK.accept(p.view(-1, V), torch.zeros(K * B, V), ictl, fctl, tok.view(-1), pos, gen, fin, out, 8, dpos, stats)
    assert out[0, 1:5].tolist() == am[:, 0].tolist() and int(pos[0]) == 5 + K + 1
    assert out[1, 1:3].tolist() == [int(am[0, 1]), int(am[1, 1])] and int(pos[1]) == 7
    assert out[2, 1:2].tolist() == [int(am[0, 2])] and int(pos[2]) == 6
    assert int(pos[3]) == 5 and int(gen[3]) == 1 and int(stats[3, 0]) == 0
    assert stats[:3, 1].tolist() == [K, 1, 0]
    assert tok[0, :3].tolist() == [int(am[K, 0]), int(am[1, 1]), int(am[0, 2])]


def test_errors(pair):
    target, draft = pair
    ids = torch.randint(3, 96, (2, 8))
    kw = dict(max_new_tokens=4)
    with pytest.raises(ValueError, match="vocab_size"):
        target.generate(ids, assistant_model=LlamaForCausalLM(_cfg(1, vocab=128), precision="32-true"), **kw)
    for K in (0, 8, 2.0):
        with pytest.raises(ValueError, match="num_assistant_tokens"):
            target.generate(ids, assistant_model=draft, num_assistant_tokens=K, **kw)
    with pytest.raises(ValueError, match="max_position_embeddings"):          # 8 + 50 + 7 > 64
        target.generate(ids, assistant_model=draft, max_new_tokens=50, num_assistant_tokens=7)
    short = LlamaForCausalLM(_cfg(1, max_pos=32), precision="32-true")
    with pytest.raises(ValueError, match="max_position_embeddings.*assistant_model"):
        target.generate(ids, assistant_model=short, max_new_tokens=20, num_assistant_tokens=5)
    ar = draft.arena
    for attr, value, msg in (("device", torch.device("cuda", 0), "device|on cuda"), ("compute_dtype", torch.bfloat16, "computes"),
                             ("param_group", object(), "FULL_SHARD")):
        old = getattr(ar, attr)
        setattr(ar, attr, value)
        try:
            with pytest.raises(ValueError, match=msg):
                target.generate(ids, assistant_model=draft, **kw)
        finally:
            setattr(ar, attr, old)
    target.arena.param_group = object()
    try:
        with pytest.raises(ValueError, match="FULL_SHARD"):
            target.generate(ids, assistant_model=draft, **kw)
    finally:
        target.arena.param_group = None


def test_cli_assistant_model(tmp_path):
    t_dir, d_dir = tmp_path / "t", tmp_path / "d"
    _cfg(2).save_pretrained(str(t_dir))
    _cfg(1).save_pretrained(str(d_dir))
    args = ["--prompt-ids", "5 17 33", "--prompt-ids", "9", "--max-new-tokens", "11", "--eos-token-id", "-1", "--init-seed", "4"]
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    run = lambda *a: subprocess.run([sys.executable, SCRIPT, "--model", str(t_dir), *args, *a], capture_output=True, text=True,  # noqa: E731
                                    env=env, cwd=ROOT)
    plain, assisted = run(), run("--assistant-model", str(d_dir), "--num-assistant-tokens", "3")
    assert plain.returncode == 0 and assisted.returncode == 0, (plain.stderr, assisted.stderr)
    assert [l for l in plain.stdout.splitlines() if l.startswith("ids:")] == \
        [l for l in assisted.stdout.splitlines() if l.startswith("ids:")]
    assert "acceptance" in assisted.stdout
