"""FP8 weight-only generation and scoring on the PyTorch reference path (CPU): the per-row quantiser reference, and
``generate`` / ``score`` with ``fp8_weights=True`` against the same calls on a copy of the model whose projection weights
were replaced by their dequantised values Ŵ, in every generation mode; re-quantisation after an in-place weight change,
untouched training state, the default path, the errors and the CLI flags."""
import json
import os
import subprocess
import sys

import pytest
import torch

from opendiloco_b200.models import fp8_weights as W8
from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import fp8 as F
from opendiloco_b200.ops import fp8w as FW

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEN = os.path.join(ROOT, "scripts", "generate.py")
EVAL = os.path.join(ROOT, "scripts", "evaluate.py")
FIRST = {"qkv": "self_attn.q_proj.weight", "o": "self_attn.o_proj.weight", "gu": "mlp.gate_proj.weight",
         "down": "mlp.down_proj.weight"}


def master_view(ar, kind, l):
    """The fp32 master rows of projection ``kind`` of layer l (q|k|v and gate|up are adjacent in the arena)."""
    N, K = W8.arena_weight(ar, kind, l).shape
    s = ar.slots[f"model.layers.{l}.{FIRST[kind]}"]
    return ar.master[s.offset:s.offset + N * K].view(N, K)


def what_copy(model):
    """A copy of ``model`` whose projection weights are Ŵ = q * inv of the per-row reference quantiser."""
    cp = LlamaForCausalLM(model.config, device=model.device, precision=model.precision, init=False)
    cp.arena.master.copy_(model.arena.master)
    cp.arena.sync_shadow()
    for kind in W8.KINDS:
        for l in range(model.config.num_hidden_layers):
            q, inv = FW.quantize_rows_ref(W8.arena_weight(model.arena, kind, l))
            master_view(cp.arena, kind, l).copy_(FW.dequantize_rows(q, inv, torch.float32))
    cp.arena.sync_shadow()
    return cp


def _prompts(V, B=3, P=10, seed=0):
    ids = torch.randint(3, V, (B, P), generator=torch.Generator().manual_seed(seed))
    mask = torch.ones_like(ids)
    mask[1, :4] = 0
    return ids.masked_fill(mask == 0, 0), mask


@pytest.fixture(scope="module")
def golden(ref_model_dir):
    m = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    return m, what_copy(m)


# ------------------------------------------------------------------------------------------------ quantiser reference
def _rows():
    g = torch.Generator().manual_seed(3)
    w = torch.randn(8, 64, generator=g) * 0.02
    w[1] = 0.0                                        # all-zero row: scale 1, q = 0
    w[2] = torch.linspace(-2.0, 2.0, 64)              # amax exactly 2: scale 2^7, +-2 -> +-256
    w[3] = torch.linspace(-3.5, 3.5, 64)              # amax 3.5: scale 2^7, +-3.5 -> +-448 (the e4m3 maximum)
    w[4, 5] = 447.99                                  # amax just under 448: scale 1, rounds onto +448
    w[5] = torch.randn(64, generator=g) * 1e-30       # tiny row: a large scale
    w[6, 7] = float("nan")                            # NaN row
    return w.to(torch.bfloat16)


def test_row_quantizer_reference():
    w = _rows()
    q, inv = FW.quantize_rows_ref(w)
    qb = q.view(torch.uint8)
    fin = ~torch.isnan(inv)
    assert fin.tolist() == [True] * 6 + [False, True]
    # power-of-two scales, 1 for the zero row, 448 <= amax * scale < 896 otherwise
    s = 1.0 / inv[fin]
    assert torch.equal(torch.frexp(s).mantissa, torch.full_like(s, 0.5))
    assert float(inv[1]) == 1.0 and torch.equal(qb[1], torch.zeros_like(qb[1]))
    assert float(inv[2]) == 2.0 ** -7 and float(q[2].float().abs().max()) == 256.0
    assert float(inv[3]) == 2.0 ** -7 and float(q[3].float().max()) == 448.0 and float(q[3].float().min()) == -448.0
    assert float(inv[4]) == 1.0 and float(q[4, 5].float()) == 448.0
    assert float(inv[5]) < 2.0 ** -90
    amax = w.float().abs().amax(dim=1)
    ok = fin & (amax > 0)
    assert bool(((amax[ok] / inv[ok]) <= 448).all()) and bool(((amax[ok] / inv[ok]) > 224).all())
    # saturating: no NaN byte in a finite row; the NaN row is all NaN bytes
    assert not bool(((qb[fin] & 0x7F) == 0x7F).any())
    assert torch.equal(qb[6], torch.full_like(qb[6], 0x7F))
    # Ŵ = q * inv exactly, and a bf16 number
    d = FW.dequantize_rows(q, inv)
    assert d.dtype == torch.bfloat16
    assert torch.equal(d[fin].float(), q[fin].float() * inv[fin, None])
    assert bool(torch.isnan(d[6]).all())
    # every row equals the per-tensor reference applied to that row alone
    for r in range(w.shape[0]):
        qr, ir = F.quantize_ref(w[r:r + 1], F.E4M3)
        assert torch.equal(qr.view(torch.uint8), qb[r:r + 1])
        assert torch.equal(ir, inv[r:r + 1]) or (torch.isnan(ir).all() and torch.isnan(inv[r]))
        dr = F.dequantize(qr, ir)
        assert torch.equal(dr.isnan(), d[r:r + 1].isnan())
        assert torch.equal(dr.nan_to_num(), d[r:r + 1].nan_to_num())


def test_fp8_state_holds_the_reference(golden):
    m, _ = golden
    fw = W8.fp8_weights(m)
    assert m.engine.fp8_weights is fw and not fw.kernels
    for kind in W8.KINDS:
        for l in range(m.config.num_hidden_layers):
            q, inv = FW.quantize_rows_ref(W8.arena_weight(m.arena, kind, l))
            assert torch.equal(fw.q[kind][l].view(torch.uint8), q.view(torch.uint8))
            assert torch.equal(fw.inv[kind][l], inv)
            assert torch.equal(fw.weight(kind, l), FW.dequantize_rows(q, inv, torch.float32))


# ------------------------------------------------------------------------------------------------ generate / score
@pytest.mark.parametrize("mode", ["greedy", "sample", "beam", "lookup", "processors", "assisted"])
def test_generate_equals_what_model(golden, mode):
    m, cp = golden
    ids, mask = _prompts(m.config.vocab_size)
    kw = {"greedy": {}, "sample": {"do_sample": True, "top_k": 20, "top_p": 0.9, "temperature": 0.8, "seed": 11},
          "beam": {"num_beams": 3, "num_return_sequences": 2, "return_dict_in_generate": True},
          "lookup": {"prompt_lookup_num_tokens": 3},
          "processors": {"repetition_penalty": 1.3, "no_repeat_ngram_size": 2, "min_new_tokens": 5}}.get(mode, {})
    if mode == "assisted":                            # only the target is quantised: the draft is the bf16-weight model
        got = m.generate(ids, attention_mask=mask, max_new_tokens=12, assistant_model=m, fp8_weights=True)
        ref = cp.generate(ids, attention_mask=mask, max_new_tokens=12, assistant_model=m)
    else:
        got = m.generate(ids, attention_mask=mask, max_new_tokens=12, fp8_weights=True, **kw)
        ref = cp.generate(ids, attention_mask=mask, max_new_tokens=12, **kw)
    if mode == "beam":
        assert torch.equal(got.sequences, ref.sequences)
        assert torch.allclose(got.sequences_scores, ref.sequences_scores, atol=1e-6, rtol=0)
    else:
        assert torch.equal(got, ref)


def test_generate_differs_from_unquantised(golden):
    """The option does something: the quantised model's logits are not the original ones."""
    m, cp = golden
    ids, _ = _prompts(m.config.vocab_size)
    assert not torch.equal(m.score(ids).logprobs, cp.score(ids).logprobs)


def test_score_equals_what_model(golden):
    m, cp = golden
    ids, mask = _prompts(m.config.vocab_size, B=4, P=17, seed=2)
    got = m.score(ids, attention_mask=mask, fp8_weights=True)
    ref = cp.score(ids, attention_mask=mask)
    assert torch.equal(got.logprobs, ref.logprobs) and torch.equal(got.greedy, ref.greedy)


def test_60m_shape_greedy_and_beam():
    cfg = LlamaConfig.from_pretrained("60m")
    cfg.vocab_size = 512
    m = LlamaForCausalLM(cfg, precision="32-true", seed=1)
    cp = what_copy(m)
    ids, mask = _prompts(cfg.vocab_size, B=2, P=6, seed=4)
    assert torch.equal(m.generate(ids, attention_mask=mask, max_new_tokens=6, fp8_weights=True),
                       cp.generate(ids, attention_mask=mask, max_new_tokens=6))
    got = m.generate(ids, attention_mask=mask, max_new_tokens=5, num_beams=2, return_dict_in_generate=True, fp8_weights=True)
    ref = cp.generate(ids, attention_mask=mask, max_new_tokens=5, num_beams=2, return_dict_in_generate=True)
    assert torch.equal(got.sequences, ref.sequences)
    assert torch.allclose(got.sequences_scores, ref.sequences_scores, atol=1e-6, rtol=0)


def test_requantises_after_in_place_change(ref_model_dir):
    m = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    ids, _ = _prompts(m.config.vocab_size)
    first = m.score(ids, fp8_weights=True).logprobs
    buffers = {k: m.engine.fp8_weights.q[k].data_ptr() for k in W8.KINDS}
    with torch.no_grad():                              # an optimizer-like in-place update of every projection
        for kind in W8.KINDS:
            for l in range(m.config.num_hidden_layers):
                v = master_view(m.arena, kind, l)
                v.add_(torch.randn(v.shape, generator=torch.Generator().manual_seed(l)) * 0.01)
        m.arena.sync_shadow()
    assert m.arena.version == 0
    second = m.score(ids, fp8_weights=True).logprobs
    assert {k: m.engine.fp8_weights.q[k].data_ptr() for k in W8.KINDS} == buffers     # same buffers, new contents
    assert not torch.equal(first, second)
    assert torch.equal(second, what_copy(m).score(ids).logprobs)
    assert torch.equal(m.generate(ids, max_new_tokens=8, fp8_weights=True), what_copy(m).generate(ids, max_new_tokens=8))


def test_training_state_untouched(ref_model_dir):
    m = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="bf16-mixed")
    ids, mask = _prompts(m.config.vocab_size)
    m.forward_backward(ids, ids)                       # a workspace and gradients to compare
    opt = torch.optim.AdamW(m.parameters(), lr=1e-3)
    opt.step()
    m.sync_compute_weights()
    before = {n: t.clone() for n, t in (("master", m.arena.master), ("shadow", m.arena.shadow), ("grad", m.arena.grad))}
    state = {id(p): {k: v.clone() for k, v in opt.state[p].items()} for p in m.parameters() if p in opt.state}
    ws = dict(m.engine._ws)
    m.generate(ids, attention_mask=mask, max_new_tokens=6, fp8_weights=True)
    m.score(ids, fp8_weights=True)
    for n, t in before.items():
        assert torch.equal(getattr(m.arena, n).view(torch.uint8), t.view(torch.uint8)), n
    for p in m.parameters():
        if p in opt.state:
            for k, v in opt.state[p].items():
                assert torch.equal(v, state[id(p)][k])
    assert m.engine._ws == ws


def test_default_path_unchanged(ref_model_dir):
    m = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    ids, mask = _prompts(m.config.vocab_size)
    a = m.generate(ids, attention_mask=mask, max_new_tokens=10)
    b = m.generate(ids, attention_mask=mask, max_new_tokens=10, fp8_weights=False)
    s = m.score(ids).logprobs
    assert torch.equal(a, b) and torch.equal(s, m.score(ids, fp8_weights=False).logprobs)
    assert m.engine.fp8_weights is None                # nothing was quantised or allocated
    m.generate(ids, max_new_tokens=4, fp8_weights=True)
    assert torch.equal(m.generate(ids, attention_mask=mask, max_new_tokens=10), a)     # and switching back is the bf16 model


@pytest.mark.parametrize("bad", [1, 0, "yes", None, 1.0])
def test_errors(golden, bad):
    m, _ = golden
    ids, _ = _prompts(m.config.vocab_size)
    with pytest.raises(ValueError, match="fp8_weights"):
        m.generate(ids, max_new_tokens=2, fp8_weights=bad)
    with pytest.raises(ValueError, match="fp8_weights"):
        m.score(ids, fp8_weights=bad)


def _env():
    return {**os.environ, "PYTHONPATH": ROOT + os.pathsep + os.environ.get("PYTHONPATH", "")}


def test_cli_generate_flag(golden, ref_model_dir):
    m, _ = golden
    ids = [5, 9, 17, 33, 2]
    run = subprocess.run([sys.executable, GEN, "--model", ref_model_dir, "--device", "cpu", "--prompt-ids", " ".join(map(str, ids)),
                          "--max-new-tokens", "8", "--eos-token-id", "-1", "--fp8-weights"],
                         capture_output=True, text=True, env=_env(), cwd=ROOT)
    assert run.returncode == 0, run.stderr
    line = [x for x in run.stdout.splitlines() if x.startswith("ids:")][0]
    want = m.generate(torch.tensor([ids]), max_new_tokens=8, eos_token_id=-1, fp8_weights=True)[0].tolist()
    assert [int(t) for t in line.split()[1:]] == want


def test_cli_evaluate_flag(golden, ref_model_dir, tmp_path):
    from opendiloco_b200.utils.data import TokenFileLoader, write_token_shard

    m, cp = golden
    write_token_shard(str(tmp_path / "val.tok"), torch.randint(0, m.config.vocab_size, (2048,), generator=torch.Generator().manual_seed(1)))
    args = [sys.executable, EVAL, "--model", ref_model_dir, "--device", "cpu", "--tokens", str(tmp_path / "*.tok"), "--seq-len", "32",
            "--batch-size", "2", "--batches", "2", "--seed", "3"]
    runs = [subprocess.run(args + extra, capture_output=True, text=True, env=_env(), cwd=ROOT) for extra in ([], ["--fp8-weights"])]
    for r in runs:
        assert r.returncode == 0, r.stderr
    plain, fp8 = (json.loads(r.stdout.strip().splitlines()[-1]) for r in runs)
    assert "fp8_weights" not in plain and fp8["fp8_weights"] is True
    loader = TokenFileLoader(str(tmp_path / "*.tok"), 2, 32, seed=3, pin_memory=False)
    nll = 0.0
    for _ in range(2):
        nll -= float(cp.score(next(loader)["input_ids"].clone()).logprobs[:, 1:].double().sum())
    loader.close()
    assert abs(fp8["loss"] - nll / fp8["tokens"]) < 1e-6
    assert fp8["loss"] != plain["loss"]
