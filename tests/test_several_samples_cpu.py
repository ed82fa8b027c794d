"""Multi-sample generation (``generate(do_sample=True, num_return_sequences=n)``) on the PyTorch reference path.

The oracle is the repeated-prompt program: ``generate(ids.repeat_interleave(n, 0), attention_mask=mask.repeat_interleave(n,
0), ...)`` with the same other arguments, which must give exactly the same tokens.  Covered: n 1, 2 and 5 on a small fp32
model and on the golden 2m, left padding with unequal lengths (one prompt of exactly 128 tokens), EOS hit early, the
warpers, each logits processor, FP8 weights, the FP8 cache and ``return_dict_in_generate``.  Also: the fork reference on
ragged lengths, every error, the unchanged default call and the CLI flag."""
import os
import subprocess
import sys

import pytest
import torch

from opendiloco_b200.models import generation as GEN
from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import decode as DK

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEN_SCRIPT = os.path.join(ROOT, "scripts", "generate.py")


@pytest.fixture(scope="module")
def golden(ref_model_dir):
    return LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")


@pytest.fixture(scope="module")
def small():
    cfg = LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
                      vocab_size=96, max_position_embeddings=256)
    return LlamaForCausalLM(cfg, precision="32-true", seed=1)


def _prompts(V, B=3, P=10, seed=0):
    ids = torch.randint(3, V, (B, P), generator=torch.Generator().manual_seed(seed))
    mask = torch.ones_like(ids)
    mask[1, :4] = 0
    mask[B - 1, :1] = 0
    return ids, mask


def _repeated(model, ids, mask, n, **kw):
    return model.generate(ids.repeat_interleave(n, 0), attention_mask=mask.repeat_interleave(n, 0), **kw)


def _same(got, ref):
    if isinstance(ref, GEN.GenerateOutput):
        assert isinstance(got, GEN.GenerateOutput) and got.sequences_scores is None and ref.sequences_scores is None
        got, ref = got.sequences, ref.sequences
    assert got.shape == ref.shape
    assert torch.equal(got, ref)


MODES = {"plain": {},
         "warpers": {"temperature": 0.7, "top_k": 20, "top_p": 0.9},
         "eos": {"pad_token_id": 1, "temperature": 1.5},
         "penalty": {"repetition_penalty": 1.3},
         "ngram": {"no_repeat_ngram_size": 2},
         "min_new": {"min_new_tokens": 6, "eos_token_id": [5, 9, 13]},
         "fp8_weights": {"fp8_weights": True},
         "fp8_kv_cache": {"fp8_kv_cache": True},
         "dict": {"return_dict_in_generate": True, "top_p": 0.8}}


@pytest.mark.parametrize("n", [1, 2, 5])
@pytest.mark.parametrize("mode", list(MODES))
def test_golden_equals_repeated_program(golden, mode, n):
    ids, mask = _prompts(golden.config.vocab_size)
    kw = dict(MODES[mode], max_new_tokens=12, do_sample=True, seed=7)
    kw.setdefault("eos_token_id", [])
    if mode == "eos":                                 # EOS ids that stop rows early: tokens the rows draw at step 2 without EOS
        kw["eos_token_id"] = sorted(set(_repeated(golden, ids, mask, n, **kw)[:, ids.shape[1] + 2].tolist()))[:8]
    got = golden.generate(ids, attention_mask=mask, num_return_sequences=n, **kw)
    _same(got, _repeated(golden, ids, mask, n, **kw))
    if mode == "eos":
        assert bool((got[:, -1] == 1).any())          # a row stopped early and was padded


@pytest.mark.parametrize("n", [2, 5])
def test_small_model_long_prompts(small, n):
    """Prompt lengths 128 (a complete chunk), 129 and 40 in one left-padded batch."""
    ids = torch.randint(3, small.config.vocab_size, (3, 129), generator=torch.Generator().manual_seed(2))
    mask = torch.ones_like(ids)
    mask[0, :1] = 0
    mask[2, :89] = 0
    kw = dict(max_new_tokens=10, do_sample=True, seed=3, temperature=0.9, eos_token_id=[7], repetition_penalty=1.2)
    _same(small.generate(ids, attention_mask=mask, num_return_sequences=n, **kw), _repeated(small, ids, mask, n, **kw))


def test_samples_differ(golden):
    ids, mask = _prompts(golden.config.vocab_size, B=2)
    out = golden.generate(ids, attention_mask=mask, max_new_tokens=12, do_sample=True, num_return_sequences=4, eos_token_id=[])
    assert out.shape == (8, 22)
    assert torch.equal(out[:, :10], ids.repeat_interleave(4, 0))
    assert len({tuple(r) for r in out[:4, 10:].tolist()}) > 1


def test_default_call_unchanged(golden):
    ids, mask = _prompts(golden.config.vocab_size)
    kw = dict(max_new_tokens=8, do_sample=True, seed=5, eos_token_id=[])
    a = golden.generate(ids, attention_mask=mask, **kw)
    st = golden.engine.decode_state
    assert st.group == 1 and st.table is None and st.B == 3
    assert torch.equal(a, golden.generate(ids, attention_mask=mask, num_return_sequences=1, **kw))
    golden.generate(ids, attention_mask=mask, num_return_sequences=2, **kw)
    assert golden.engine.decode_state.group == 2 and golden.engine.decode_state.B == 6
    assert torch.equal(a, golden.generate(ids, attention_mask=mask, **kw))
    assert golden.engine.decode_state.group == 1


def test_fork_reference_ragged():
    L, rows, Hkv, Smax, D, n = 2, 6, 2, 384, 4, 3
    kv = torch.randn(L, 2, rows, Hkv, Smax, D)
    inv = torch.randn(L, 2, rows, Hkv, Smax)
    before, before_inv = kv.clone(), inv.clone()
    DK.fork(kv, None, torch.tensor([128, 129], dtype=torch.int32), n, inv=inv)
    src = torch.tensor([0, 0, 0, 3, 3, 3])
    assert torch.equal(kv, before[:, :, src]) and torch.equal(inv, before_inv[:, :, src])


def test_errors(golden):
    ids, mask = _prompts(golden.config.vocab_size)
    for r in (0, -1, 2.0, True, "2"):
        with pytest.raises(ValueError, match="num_return_sequences"):
            golden.generate(ids, max_new_tokens=2, do_sample=True, num_return_sequences=r)
    with pytest.raises(ValueError, match="num_return_sequences"):
        golden.generate(ids, max_new_tokens=2, num_return_sequences=2)
    with pytest.raises(ValueError, match="num_return_sequences"):
        golden.generate(ids, max_new_tokens=2, do_sample=True, num_return_sequences=2, assistant_model=golden)
    with pytest.raises(ValueError, match="num_return_sequences"):
        golden.generate(ids, max_new_tokens=2, do_sample=True, num_return_sequences=2, prompt_lookup_num_tokens=3)
    with pytest.raises(ValueError, match="num_return_sequences"):
        golden.generate(ids, max_new_tokens=2, num_beams=2, num_return_sequences=3)


def test_cli_flag(golden, ref_model_dir):
    prompts = [[5, 9, 17, 33, 2], [7, 8]]
    env = {**os.environ, "PYTHONPATH": ROOT + os.pathsep + os.environ.get("PYTHONPATH", "")}
    args = [sys.executable, GEN_SCRIPT, "--model", ref_model_dir, "--device", "cpu", "--max-new-tokens", "6", "--eos-token-id", "-1",
            "--do-sample", "--seed", "4", "--num-return-sequences", "3"]
    for p in prompts:
        args += ["--prompt-ids", " ".join(map(str, p))]
    run = subprocess.run(args, capture_output=True, text=True, env=env, cwd=ROOT)
    assert run.returncode == 0, run.stderr
    lines = [[int(t) for t in x.split()[1:]] for x in run.stdout.splitlines() if x.startswith("ids:")]
    ids = torch.tensor([prompts[0], [0, 0, 0] + prompts[1]])                # the script's left padding
    mask = torch.tensor([[1] * 5, [0, 0, 0, 1, 1]])
    want = golden.generate(ids, attention_mask=mask, max_new_tokens=6, eos_token_id=-1, do_sample=True, seed=4, num_return_sequences=3)
    assert len(lines) == 6
    for i, row in enumerate(lines):
        p = prompts[i // 3]
        assert row == p + want[i, 5:].tolist()
