"""Beam search (``generate(num_beams=...)``) on the PyTorch reference path (CPU): parity with transformers' beam search,
the chunk-table attention reference, argument errors and the command-line front-end."""
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
PAD = 7
N_NEW = 14


def _batch(V, padded, P=9, seed=0):
    ids = torch.randint(3, V, (3, P), generator=torch.Generator().manual_seed(seed))
    mask = torch.ones_like(ids)
    if padded:
        mask[1, :3] = 0
        mask[2, :5] = 0
    return ids.masked_fill(mask == 0, 0), mask


@pytest.fixture(scope="module")
def models(ref_model_dir):
    tr = pytest.importorskip("transformers")
    ours = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    hf = tr.LlamaForCausalLM.from_pretrained(ref_model_dir, attn_implementation="sdpa").float().eval()
    return ours, hf


@pytest.fixture(scope="module")
def early_tokens(models):
    """Tokens the model emits early in its beams (no EOS): EOS ids that end hypotheses at different lengths."""
    ours, _ = models
    ids, mask = _batch(ours.config.vocab_size, True)
    out = ours.generate(ids, attention_mask=mask, max_new_tokens=6, num_beams=4, num_return_sequences=4, eos_token_id=[])
    new = out[:, ids.shape[1]:]
    picks = []
    for t in new[:, 1:].flatten().tolist() + new[:, 0].tolist():
        if t not in picks:
            picks.append(t)
    return picks


def _compare(models, padded, eos, **kw):
    ours, hf = models
    ids, mask = _batch(ours.config.vocab_size, padded)
    got = ours.generate(ids, attention_mask=mask, max_new_tokens=N_NEW, eos_token_id=eos, pad_token_id=PAD,
                        return_dict_in_generate=True, **kw)
    with torch.no_grad():
        ref = hf.generate(ids, attention_mask=mask, max_new_tokens=N_NEW, do_sample=False, eos_token_id=eos, pad_token_id=PAD,
                          output_scores=True, return_dict_in_generate=True, **kw)
    seq = ref.sequences
    seq = torch.cat([seq, torch.full((seq.shape[0], got.sequences.shape[1] - seq.shape[1]), PAD)], dim=1)
    R = kw.get("num_return_sequences", 1)
    assert got.sequences.shape == (ids.shape[0] * R, ids.shape[1] + N_NEW)
    assert torch.equal(got.sequences, seq), (got.sequences, seq)
    assert torch.allclose(got.sequences_scores, ref.sequences_scores.float(), atol=1e-5, rtol=0)
    return got


@pytest.mark.parametrize("num_beams", [2, 4, 8])
@pytest.mark.parametrize("all_returned", [False, True])
@pytest.mark.parametrize("padded", [False, True])
def test_matches_hf_beam_search(models, early_tokens, num_beams, all_returned, padded):
    got = _compare(models, padded, early_tokens[0], num_beams=num_beams, num_return_sequences=num_beams if all_returned else 1)
    assert got.sequences_scores.dtype == torch.float32


@pytest.mark.parametrize("length_penalty", [1.0, 0.0, 2.0, -0.5])
@pytest.mark.parametrize("early_stopping", [False, True, "never"])
def test_matches_hf_length_penalty_and_early_stopping(models, early_tokens, length_penalty, early_stopping):
    _compare(models, True, early_tokens[:3], num_beams=4, num_return_sequences=4, length_penalty=length_penalty,
             early_stopping=early_stopping)


def test_hypotheses_finish_at_different_lengths(models, early_tokens):
    got = _compare(models, True, early_tokens[:4], num_beams=4, num_return_sequences=4)
    P = 9
    new = got.sequences[:, P:]
    lengths = {int((row != PAD).sum()) for row in new}
    assert len(lengths) > 1, lengths                   # the EOS ids really end hypotheses early


def test_num_beams_1_is_todays_generate(models):
    ours, _ = models
    ids, mask = _batch(ours.config.vocab_size, True)
    plain = ours.generate(ids, attention_mask=mask, max_new_tokens=10)
    assert torch.equal(ours.generate(ids, attention_mask=mask, max_new_tokens=10, num_beams=1), plain)
    res = ours.generate(ids, attention_mask=mask, max_new_tokens=10, num_beams=1, return_dict_in_generate=True)
    assert torch.equal(res.sequences, plain) and res.sequences_scores is None


def test_last_step_stays_inside_the_cache(models):
    """P + max_new_tokens a multiple of 128: every position written or reordered stays below Smax."""
    ours, _ = models
    ids, mask = _batch(ours.config.vocab_size, False)
    n_new = 128 - ids.shape[1]
    ours.generate(ids, attention_mask=mask, max_new_tokens=n_new, num_beams=4, eos_token_id=[])
    bs = ours.engine.beam_state
    assert int(bs.dec.pos.max()) == ids.shape[1] + n_new - 1 == bs.dec.Smax - 1


def test_table_attention_reference_equals_reordered_cache():
    g = torch.Generator().manual_seed(0)
    rows, Hq, Hkv, D, Smax = 6, 4, 2, 64, 512
    nch = Smax // 128
    q = torch.randn(rows, (Hq + 2 * Hkv) * D, generator=g)
    kc, vc = torch.randn(rows, Hkv, Smax, D, generator=g), torch.randn(rows, Hkv, Smax, D, generator=g)
    table = torch.randint(0, rows, (rows, nch), generator=g, dtype=torch.int64).int()
    pos = torch.tensor([0, 127, 128, 300, 383, 511], dtype=torch.int32)
    got = torch.empty(rows, Hq * D)
    DK.attention(q, kc, vc, pos, got, Hq, Hkv, D, table=table)
    kg, vg = torch.empty_like(kc), torch.empty_like(vc)
    for r in range(rows):
        for c in range(nch):
            src = int(table[r, c])
            kg[r, :, c * 128:(c + 1) * 128] = kc[src, :, c * 128:(c + 1) * 128]
            vg[r, :, c * 128:(c + 1) * 128] = vc[src, :, c * 128:(c + 1) * 128]
    ref = torch.empty(rows, Hq * D)
    DK.attention(q, kg, vg, pos, ref, Hq, Hkv, D)
    assert torch.equal(got, ref)


def test_reorder_reference_moves_whole_rows():
    kv = torch.arange(2 * 2 * 4 * 3, dtype=torch.float32).view(2, 2, 4, 3, 1).expand(2, 2, 4, 3, 5).contiguous()
    parent = torch.tensor([1, 0, 0, 3], dtype=torch.int32)                  # a swap, a copy and a row that keeps itself
    before = kv.clone()
    DK.beam_reorder(kv, None, parent, torch.zeros(4, dtype=torch.int32), 4)
    assert torch.equal(kv, before[:, :, parent.long()])


def test_errors():
    cfg = LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2, vocab_size=96,
                      max_position_embeddings=64)
    model = LlamaForCausalLM(cfg, precision="32-true", seed=1)
    ids = torch.randint(3, cfg.vocab_size, (2, 8))
    for nb in (0, 9, 2.0, True):
        with pytest.raises(ValueError, match="num_beams"):
            model.generate(ids, max_new_tokens=2, num_beams=nb)
    for r in (0, 5):
        with pytest.raises(ValueError, match="num_return_sequences"):
            model.generate(ids, max_new_tokens=2, num_beams=4, num_return_sequences=r)
    with pytest.raises(ValueError, match="num_return_sequences"):
        model.generate(ids, max_new_tokens=2, num_return_sequences=2)
    with pytest.raises(ValueError, match="do_sample"):
        model.generate(ids, max_new_tokens=2, num_beams=2, do_sample=True)
    with pytest.raises(ValueError, match="assistant_model"):
        model.generate(ids, max_new_tokens=2, num_beams=2, assistant_model=model)
    for es in ("always", 1, None):
        with pytest.raises(ValueError, match="early_stopping"):
            model.generate(ids, max_new_tokens=2, num_beams=2, early_stopping=es)
    with pytest.raises(ValueError, match="max_position_embeddings"):
        model.generate(ids, max_new_tokens=cfg.max_position_embeddings - 7, num_beams=2)
    bad = torch.ones_like(ids)
    bad[0, -1] = 0
    with pytest.raises(ValueError, match="left-padded"):
        model.generate(ids, attention_mask=bad, max_new_tokens=2, num_beams=2)
    model.arena.param_group = object()                   # what enable_param_sharding (FULL_SHARD) leaves behind
    try:
        with pytest.raises(ValueError, match="FULL_SHARD"):
            model.generate(ids, max_new_tokens=2, num_beams=2)
    finally:
        model.arena.param_group = None


def test_cli_beam_search_on_golden_model(ref_model_dir):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, SCRIPT, "--model", ref_model_dir, "--prompt-ids", "1 450 37 99", "--prompt-ids", "1 7",
                          "--max-new-tokens", "8", "--num-beams", "4", "--num-return-sequences", "2", "--length-penalty", "0.5",
                          "--early-stopping", "never"], capture_output=True, text=True, env=env, cwd=ROOT)
    assert res.returncode == 0, res.stderr
    lines = res.stdout.splitlines()
    rows = [[int(t) for t in line.split()[1:]] for line in lines if line.startswith("ids:")]
    scores = [float(line.split()[1]) for line in lines if line.startswith("score:")]
    model = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    ids = torch.tensor([[1, 450, 37, 99], [0, 0, 1, 7]])
    mask = torch.tensor([[1, 1, 1, 1], [0, 0, 1, 1]])
    out = model.generate(ids, attention_mask=mask, max_new_tokens=8, num_beams=4, num_return_sequences=2, length_penalty=0.5,
                         early_stopping="never", return_dict_in_generate=True)
    assert len(rows) == 4 and len(scores) == 4
    assert rows[0] == out.sequences[0].tolist() and rows[1] == out.sequences[1].tolist()
    assert rows[2] == out.sequences[2, 2:].tolist() and rows[3] == out.sequences[3, 2:].tolist()
    assert scores == pytest.approx(out.sequences_scores.tolist(), abs=1e-6)
