"""KV-cached generation on the PyTorch reference path (CPU): parity with transformers and with our own full forward,
output rules, argument errors and the command-line front-end."""
import os
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch

from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.generation import decode_state, prefill, step
from opendiloco_b200.models.llama import LlamaForCausalLM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "scripts", "generate.py")


def _ragged_batch(V, P=9, seed=0):
    ids = torch.randint(3, V, (3, P), generator=torch.Generator().manual_seed(seed))
    mask = torch.ones_like(ids)
    mask[1, :3] = 0
    mask[2, :5] = 0
    return ids.masked_fill(mask == 0, 0), mask


def _tiny_cfg():
    return LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2, vocab_size=96,
                       max_position_embeddings=64)


@pytest.mark.parametrize("padded", [False, True])
def test_greedy_matches_hf_generate(ref_model_dir, padded):
    tr = pytest.importorskip("transformers")
    ours = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    hf = tr.LlamaForCausalLM.from_pretrained(ref_model_dir, attn_implementation="sdpa").float().eval()
    ids, mask = _ragged_batch(ours.config.vocab_size)
    if not padded:
        mask = torch.ones_like(mask)
    n_new = 24
    got = ours.generate(ids, attention_mask=mask, max_new_tokens=n_new)
    with torch.no_grad():
        ref = hf.generate(ids, attention_mask=mask, max_new_tokens=n_new, do_sample=False, pad_token_id=2, output_logits=True,
                          return_dict_in_generate=True)
    seq, logits = ref.sequences, torch.stack(ref.logits, dim=1)       # [B, steps, V]
    assert got.shape == (ids.shape[0], ids.shape[1] + n_new)
    assert torch.equal(got[:, : ids.shape[1]], ids)
    P = ids.shape[1]
    for b in range(ids.shape[0]):
        for t in range(seq.shape[1] - P):
            if got[b, P + t] != seq[b, P + t]:
                top2 = logits[b, t].topk(2).values
                gap = float(top2[0] - top2[1])
                print(f"row {b} step {t}: ours {int(got[b, P + t])} vs HF {int(seq[b, P + t])}, HF top-two gap {gap:.3g}")
                assert gap < 1e-4
                break                                    # the continuations differ from here on
    if seq.shape[1] < got.shape[1]:                      # HF stopped early: every row had finished
        assert bool((got[:, seq.shape[1]:] == 2).all())


def test_teacher_forced_decode_logits_match_full_forward(ref_model_dir):
    model = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    V = model.config.vocab_size
    B, P, n = 2, 7, 10
    full = torch.randint(3, V, (B, P + n), generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        ref = model(full).logits                         # [B, P + n, V]
    st = decode_state(model, B, 64)
    st.set_controls(False, 1.0, 0, 1.0, 0, 0, [])
    prefill(model, st, full[:, :P], torch.full((B,), P, dtype=torch.int32))
    assert torch.allclose(st.logits, ref[:, P - 1], atol=1e-5, rtol=0)
    for t in range(n - 1):
        st.ids.copy_(full[:, P + t])                     # teacher forcing: feed the true next token
        step(model, st)
        err = (st.logits - ref[:, P + t]).abs().max().item()
        assert err < 1e-5, (t, err)


def test_output_rules_eos_pad_seed_topk1():
    torch.manual_seed(0)
    cfg = _tiny_cfg()
    model = LlamaForCausalLM(cfg, precision="32-true", seed=1)
    ids, mask = _ragged_batch(cfg.vocab_size, P=6, seed=2)
    greedy = model.generate(ids, attention_mask=mask, max_new_tokens=12, eos_token_id=[])
    assert greedy.shape == (3, 18) and greedy.dtype == torch.int64
    assert torch.equal(greedy[:, :6], ids)
    # EOS: make the second greedy token of row 0 the EOS id -> everything after it is pad
    eos = int(greedy[0, 7])
    out = model.generate(ids, attention_mask=mask, max_new_tokens=12, eos_token_id=eos, pad_token_id=95)
    for b in range(3):
        new = out[b, 6:].tolist()
        if eos in new:
            k = new.index(eos)
            assert all(t == 95 for t in new[k + 1:]), new
            assert new[: k + 1] == greedy[b, 6:6 + k + 1].tolist()
        else:
            assert new == greedy[b, 6:].tolist()
    assert out[0, 7] == eos
    # pad defaults to the EOS id
    out2 = model.generate(ids, attention_mask=mask, max_new_tokens=12, eos_token_id=eos)
    assert torch.equal(out2, torch.where(out == 95, torch.full_like(out, eos), out))
    # sampling: a fixed seed reproduces; top_k=1 is greedy
    kw = dict(attention_mask=mask, max_new_tokens=12, do_sample=True, temperature=1.3, top_k=0, eos_token_id=[])
    s1, s2 = model.generate(ids, seed=5, **kw), model.generate(ids, seed=5, **kw)
    assert torch.equal(s1, s2)
    assert not torch.equal(s1, model.generate(ids, seed=6, **kw))
    assert torch.equal(model.generate(ids, attention_mask=mask, max_new_tokens=12, do_sample=True, top_k=1, eos_token_id=[]), greedy)


def test_errors():
    cfg = _tiny_cfg()
    model = LlamaForCausalLM(cfg, precision="32-true", seed=1)
    ids = torch.randint(3, cfg.vocab_size, (2, 8))
    with pytest.raises(ValueError, match="max_position_embeddings"):
        model.generate(ids, max_new_tokens=cfg.max_position_embeddings - 7)
    bad = torch.ones_like(ids)
    bad[0, -1] = 0                                       # right padding
    with pytest.raises(ValueError, match="left-padded"):
        model.generate(ids, attention_mask=bad, max_new_tokens=2)
    holes = torch.ones_like(ids)
    holes[1, 3] = 0                                      # a gap inside the prompt
    with pytest.raises(ValueError, match="left-padded"):
        model.generate(ids, attention_mask=holes, max_new_tokens=2)
    model.arena.param_group = object()                   # what enable_param_sharding (FULL_SHARD) leaves behind
    try:
        with pytest.raises(ValueError, match="FULL_SHARD"):
            model.generate(ids, max_new_tokens=2)
    finally:
        model.arena.param_group = None


def _run_cli(*args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, SCRIPT, *args], capture_output=True, text=True, env=env, cwd=ROOT)
    return res


def _cli_ids(res):
    assert res.returncode == 0, res.stderr
    return [[int(t) for t in line.split()[1:]] for line in res.stdout.splitlines() if line.startswith("ids:")]


def test_cli_on_golden_model(ref_model_dir):
    res = _run_cli("--model", ref_model_dir, "--prompt-ids", "1 450 37 99", "--prompt-ids", "1 7", "--max-new-tokens", "8")
    rows = _cli_ids(res)
    model = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    ids = torch.tensor([[1, 450, 37, 99], [0, 0, 1, 7]])
    mask = torch.tensor([[1, 1, 1, 1], [0, 0, 1, 1]])
    out = model.generate(ids, attention_mask=mask, max_new_tokens=8)
    assert rows[0] == out[0].tolist()
    assert rows[1] == out[1, 2:].tolist()


def test_cli_reads_training_checkpoint_local_and_outer(tmp_path):
    from opendiloco_b200.optim.fused import FusedAdamW
    from opendiloco_b200.utils.ckpt import save_checkpoint

    cfg = _tiny_cfg()
    cfg_dir = tmp_path / "cfg"
    cfg.save_pretrained(str(cfg_dir))
    model = LlamaForCausalLM(cfg, precision="32-true", seed=3)
    opt = FusedAdamW(model.parameters(), lr=1e-3)
    theta_outer = model.arena.master.clone()
    theta_outer += 0.05 * torch.randn(theta_outer.shape, generator=torch.Generator().manual_seed(0))
    diloco = SimpleNamespace(state_averager=SimpleNamespace(theta_outer=theta_outer, momentum_buffer=None))
    with_outer, without_outer = tmp_path / "ck_outer", tmp_path / "ck_plain"
    save_checkpoint(str(with_outer), model, opt, diloco=diloco, rank=0, save_global_state=False)
    save_checkpoint(str(without_outer), model, opt, rank=0, save_global_state=False)

    prompt = [5, 17, 33, 2, 60]
    ids = torch.tensor([prompt])
    for which, flat in (("local", model.arena.master), ("outer", theta_outer)):
        res = _run_cli("--model", str(cfg_dir), "--checkpoint", str(with_outer), "--weights", which,
                       "--prompt-ids", " ".join(map(str, prompt)), "--max-new-tokens", "10", "--eos-token-id", "-1")
        ref = LlamaForCausalLM(cfg, precision="32-true", init=False)
        ref.arena.master.copy_(flat)
        ref.arena.sync_shadow()
        assert _cli_ids(res)[0] == ref.generate(ids, max_new_tokens=10, eos_token_id=-1)[0].tolist(), which
    a = _cli_ids(_run_cli("--model", str(cfg_dir), "--checkpoint", str(with_outer), "--weights", "local", "--prompt-ids", "5 17",
                          "--max-new-tokens", "10", "--eos-token-id", "-1"))
    b = _cli_ids(_run_cli("--model", str(cfg_dir), "--checkpoint", str(with_outer), "--weights", "outer", "--prompt-ids", "5 17",
                          "--max-new-tokens", "10", "--eos-token-id", "-1"))
    assert a != b                                        # the two weight sets really are different models

    res = _run_cli("--model", str(cfg_dir), "--checkpoint", str(without_outer), "--weights", "outer", "--prompt-ids", "5 17")
    assert res.returncode != 0
    assert "no 'theta_outer' weights" in res.stderr
