"""Per-token log-likelihood scoring on the PyTorch reference path (CPU, fp32): parity with transformers and with the
model's own loss, padding, labels, argument errors and the evaluation command line."""
import json
import math
import os
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch

from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import kernels as K
from opendiloco_b200.ops import tc_gemm as TC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SCRIPT = os.path.join(ROOT, "scripts", "evaluate.py")


def _tiny_cfg():
    return LlamaConfig(hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2, vocab_size=96,
                       max_position_embeddings=64)


def _ids(V, B, S, seed):
    return torch.randint(0, V, (B, S), generator=torch.Generator().manual_seed(seed))


def test_matches_transformers_log_softmax(ref_model_dir):
    tr = pytest.importorskip("transformers")
    ours = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    hf = tr.LlamaForCausalLM.from_pretrained(ref_model_dir, attn_implementation="eager").float().eval()
    V = ours.config.vocab_size
    ids = _ids(V, 3, 150, 0)
    ids[0, 100:] = ids[0, :50]                  # a repeat the model may predict, so that some greedy flags are set
    out = ours.score(ids)
    with torch.no_grad():
        logits = hf(ids).logits.float()
    ref = torch.log_softmax(logits, dim=-1)[:, :-1].gather(2, ids[:, 1:, None])[..., 0]
    assert out.logprobs.dtype == torch.float32 and out.greedy.dtype == torch.bool and out.logprobs.shape == ids.shape
    assert (out.logprobs[:, 1:] - ref).abs().max().item() < 1e-5
    assert torch.equal(out.greedy[:, 1:], logits[:, :-1].argmax(dim=-1) == ids[:, 1:])
    assert torch.equal(out.logprobs[:, 0], torch.zeros(3)) and not out.greedy[:, 0].any()


def test_padded_batch_equals_unpadded_rows(ref_model_dir):
    model = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    S = 300
    ids = _ids(model.config.vocab_size, 4, S, 1)
    mask = torch.ones_like(ids)
    mask[0, :45] = 0                            # left padding
    mask[1, 131:] = 0                           # right padding
    mask[2, :7] = 0                             # both
    mask[2, 200:] = 0
    out = model.score(ids, attention_mask=mask)
    for b in range(4):
        cols = mask[b].nonzero()[:, 0]
        lo, hi = int(cols[0]), int(cols[-1]) + 1
        alone = model.score(ids[b:b + 1, lo:hi])
        assert (out.logprobs[b, lo:hi] - alone.logprobs[0]).abs().max().item() < 1e-6, b
        assert torch.equal(out.greedy[b, lo:hi], alone.greedy[0])
        outside = mask[b] == 0
        assert torch.equal(out.logprobs[b][outside], torch.zeros(int(outside.sum())))
        assert not out.greedy[b][outside].any()


def test_labels_ignore_index_and_position_zero():
    model = LlamaForCausalLM(_tiny_cfg(), precision="32-true", seed=0)
    ids = _ids(96, 2, 20, 2)
    labels = ids.clone()
    labels[0, 5:9] = -100
    labels[1, 12] = 3
    base = model.score(ids)
    out = model.score(ids, labels=labels)
    assert torch.equal(out.logprobs[0, 5:9], torch.zeros(4)) and not out.greedy[0, 5:9].any()
    assert torch.equal(out.logprobs[:, 0], torch.zeros(2))
    keep = labels == ids
    keep[:, 0] = False
    assert torch.equal(out.logprobs[keep], base.logprobs[keep])
    assert out.logprobs[1, 12] != base.logprobs[1, 12]
    assert bool((out.logprobs <= 1e-6).all())


def test_perplexity_matches_model_loss(ref_model_dir):
    model = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true").eval()
    ids = _ids(model.config.vocab_size, 2, 64, 3)
    with torch.no_grad():
        loss = model(ids, labels=ids).loss
    lp = model.score(ids).logprobs[:, 1:]
    assert abs(math.exp(-lp.mean().item()) - math.exp(loss.item())) < 1e-5 * math.exp(loss.item())


def test_reference_ops_planes_ties_and_range():
    """The reference pair (plane statistics + merge) against a direct logsumexp / argmax, with ties across planes and a
    vocabulary that is not a multiple of 256."""
    torch.manual_seed(0)
    T, h, V = 9, 16, 700
    x = torch.randn(T, h)
    w = torch.randn(V, h)
    w[699] = w[3] = w[300] = 4 * x[0] / x[0].norm() ** 2 * 10    # row 0: three tied maxima in three planes
    labels = torch.randint(0, V, (T,))
    labels[2] = -100
    planes = (V + 255) // 256
    pmax, psum, zlab = torch.empty(planes * T), torch.empty(planes * T), torch.empty(T)
    pidx = torch.empty(planes * T, dtype=torch.int32)
    TC.lce_score(x, w, labels, pmax, psum, pidx, zlab)
    lp, gr = torch.empty(T), torch.empty(T, dtype=torch.bool)
    lse, am = torch.empty(T), torch.empty(T, dtype=torch.int32)
    K.lce_score_finalize(pmax, psum, pidx, zlab, planes, labels, lp, gr, lse, am)
    z = x @ w.t()
    assert torch.allclose(lse, torch.logsumexp(z, dim=-1), atol=1e-5, rtol=0)
    assert torch.equal(am.long(), z.argmax(dim=-1))
    assert int(am[0]) == 3 or bool(z[0, 3] < z[0].max())              # lowest index among exact ties
    ref = z.log_softmax(dim=-1).gather(1, labels.clamp(min=0)[:, None])[:, 0]
    assert torch.allclose(lp[labels >= 0], ref[labels >= 0], atol=1e-5, rtol=0)
    assert lp[2] == 0 and not gr[2]
    assert torch.equal(gr, (labels >= 0) & (z.argmax(dim=-1) == labels))


def test_errors():
    cfg = _tiny_cfg()
    model = LlamaForCausalLM(cfg, precision="32-true", seed=1)
    ids = _ids(96, 2, 8, 4)
    with pytest.raises(ValueError, match="max_position_embeddings"):
        model.score(_ids(96, 1, cfg.max_position_embeddings + 1, 0))
    with pytest.raises(ValueError, match="input_ids must be"):
        model.score(ids[0])
    with pytest.raises(ValueError, match="attention_mask shape"):
        model.score(ids, attention_mask=torch.ones(2, 7, dtype=torch.int64))
    with pytest.raises(ValueError, match="labels shape"):
        model.score(ids, labels=ids[:, :5])
    holes = torch.ones_like(ids)
    holes[1, 3] = 0                                      # a gap inside the row
    with pytest.raises(ValueError, match="contiguous run"):
        model.score(ids, attention_mask=holes)
    with pytest.raises(ValueError, match="contiguous run"):
        model.score(ids, attention_mask=torch.zeros_like(ids))
    bad = ids.clone()
    bad[0, 2] = 96
    with pytest.raises(ValueError, match="input_ids hold token ids"):
        model.score(bad)
    lab = ids.clone()
    lab[1, 4] = -5
    with pytest.raises(ValueError, match="labels must lie"):
        model.score(ids, labels=lab)
    model.arena.param_group = object()                   # what enable_param_sharding (FULL_SHARD) leaves behind
    try:
        with pytest.raises(ValueError, match="FULL_SHARD"):
            model.score(ids)
    finally:
        model.arena.param_group = None


def test_score_leaves_training_workspaces_alone():
    model = LlamaForCausalLM(_tiny_cfg(), precision="32-true", seed=0)
    x = _ids(96, 2, 16, 5)
    model.forward_backward(x, x)
    ws = dict(model.engine._ws)
    model.score(_ids(96, 3, 11, 6))
    model.score(_ids(96, 5, 9, 7))
    assert model.engine._ws == ws
    assert model.engine.score_state is not None and model.engine.score_state.key[:3] == (5, 9, 9)


# ------------------------------------------------------------------------------------------------ command line
def _run_cli(*args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    res = subprocess.run([sys.executable, SCRIPT, *args], capture_output=True, text=True, env=env, cwd=ROOT)
    assert res.returncode == 0, res.stderr
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("{")]
    assert len(lines) == 1, res.stdout
    return json.loads(lines[0])


def test_cli_perplexity_on_token_shard(ref_model_dir, tmp_path):
    from opendiloco_b200.utils.data import TokenFileLoader, write_token_shard

    model = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    tokens = torch.randint(0, model.config.vocab_size, (4096,), generator=torch.Generator().manual_seed(8))
    write_token_shard(str(tmp_path / "val.tok"), tokens)
    got = _run_cli("--model", ref_model_dir, "--tokens", str(tmp_path / "*.tok"), "--seq-len", "64", "--batch-size", "4",
                   "--batches", "3", "--seed", "5")
    loader = TokenFileLoader(str(tmp_path / "*.tok"), 4, 64, seed=5, pin_memory=False)
    nll = 0.0
    for _ in range(3):
        ids = next(loader)["input_ids"].clone()
        nll -= float(model.score(ids).logprobs[:, 1:].double().sum())
    loader.close()
    assert got["tokens"] == 3 * 4 * 63
    assert abs(got["loss"] - nll / got["tokens"]) < 1e-6
    assert abs(got["perplexity"] - math.exp(got["loss"])) < 1e-6 * got["perplexity"]
    assert got["tokens_per_s"] > 0


def test_cli_multiple_choice_on_greedy_continuations(ref_model_dir, tmp_path):
    model = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    V = model.config.vocab_size
    g = torch.Generator().manual_seed(9)
    lines = []
    for r in range(5):
        ctx = torch.randint(3, V, (1, 4 + 3 * r), generator=g)
        n_new = 2 + r
        cont = model.generate(ctx, max_new_tokens=n_new, eos_token_id=[])[0, ctx.shape[1]:].tolist()
        others = [torch.randint(3, V, (n_new + k,), generator=g).tolist() for k in range(2)]
        gold = r % 3
        choices = others[:gold] + [cont] + others[gold:]
        lines.append(json.dumps({"context": ctx[0].tolist(), "choices": choices, "gold": gold}))
    path = tmp_path / "mc.jsonl"
    path.write_text("\n".join(lines) + "\n")
    got = _run_cli("--model", ref_model_dir, "--choices", str(path), "--batch-size", "4")
    assert got["n"] == 5
    assert got["acc"] == 1.0 and got["greedy"] == 1.0
    assert 0.0 <= got["acc_per_token"] <= 1.0


def test_cli_reads_training_checkpoint_local_and_outer(tmp_path):
    from opendiloco_b200.optim.fused import FusedAdamW
    from opendiloco_b200.utils.ckpt import save_checkpoint
    from opendiloco_b200.utils.data import write_token_shard

    cfg = _tiny_cfg()
    cfg_dir = tmp_path / "cfg"
    cfg.save_pretrained(str(cfg_dir))
    model = LlamaForCausalLM(cfg, precision="32-true", seed=3)
    opt = FusedAdamW(model.parameters(), lr=1e-3)
    theta_outer = model.arena.master.clone()
    theta_outer += 0.05 * torch.randn(theta_outer.shape, generator=torch.Generator().manual_seed(0))
    diloco = SimpleNamespace(state_averager=SimpleNamespace(theta_outer=theta_outer, momentum_buffer=None))
    ck = tmp_path / "ck"
    save_checkpoint(str(ck), model, opt, diloco=diloco, rank=0, save_global_state=False)
    write_token_shard(str(tmp_path / "val.tok"), torch.randint(0, 96, (2048,), generator=torch.Generator().manual_seed(1)))
    res = {}
    for which, flat in (("local", model.arena.master), ("outer", theta_outer)):
        res[which] = _run_cli("--model", str(cfg_dir), "--checkpoint", str(ck), "--weights", which, "--tokens",
                              str(tmp_path / "val.tok"), "--seq-len", "32", "--batch-size", "2", "--batches", "2")
        ref = LlamaForCausalLM(cfg, precision="32-true", init=False)
        ref.arena.master.copy_(flat)
        ref.arena.sync_shadow()
        from opendiloco_b200.utils.data import TokenFileLoader

        loader = TokenFileLoader(str(tmp_path / "val.tok"), 2, 32, seed=0, pin_memory=False)
        nll = -sum(float(ref.score(next(loader)["input_ids"].clone()).logprobs[:, 1:].double().sum()) for _ in range(2))
        loader.close()
        assert abs(res[which]["loss"] - nll / res[which]["tokens"]) < 1e-6, which
    assert abs(res["local"]["loss"] - res["outer"]["loss"]) > 1e-4       # the two weight sets really are different models
