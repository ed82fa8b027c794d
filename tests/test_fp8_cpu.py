"""precision="fp8-mixed" on CPU: the QDQ references of ops/fp8.py, the whole FP8 training program on those references
(loss and per-tensor gradients against bf16-mixed), the constructor's shape checks, and the training CLI."""
import os
import pickle
import socket
import subprocess
import sys

import pytest
import torch

from opendiloco_b200.models import llama as llama_mod
from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import attention as A
from opendiloco_b200.ops import fp8 as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "llama-2m-fresh")


# ------------------------------------------------------------------------------------------------ QDQ reference
@pytest.mark.parametrize("fmt", [F.E4M3, F.E5M2])
@pytest.mark.parametrize("mag", [1e-6, 0.37, 3.0, 1e4])
def test_scale_is_the_largest_power_of_two_that_fits(fmt, mag):
    x = (torch.randn(64, 128) * mag).to(torch.bfloat16)
    amax = x.float().abs().amax()
    scale, inv, finite = F.scale_ref(amax, fmt)
    s = float(scale)
    assert bool(finite) and s == 2.0 ** round(torch.log2(scale).item())
    assert float(amax) * s <= F.FP8_MAX[fmt] < float(amax) * s * 2
    assert float(inv) * s == 1.0
    q, inv2 = F.quantize_ref(x, fmt)
    assert float(inv2) == float(inv)
    assert float(q.float().abs().max()) <= F.FP8_MAX[fmt]


@pytest.mark.parametrize("fmt", [F.E4M3, F.E5M2])
def test_saturation_zero_and_dequantisation(fmt):
    m = F.FP8_MAX[fmt]
    # a scale taken from a smaller amax: values beyond FP8_MAX saturate instead of turning into NaN
    x = torch.tensor([[1.0, -1.0, 4.0, -4.0, 0.5, 0.0, 2.0, -3.0]])
    q, inv = F.quantize_ref(x, fmt, amax=torch.tensor([1.0]))
    v = q.float()
    assert float(v.max()) == m and float(v.min()) == -m and not torch.isnan(v).any()
    # amax = 0: scale 1, all zeros
    z, inv0 = F.quantize_ref(torch.zeros(4, 8), fmt)
    assert float(inv0) == 1.0 and (z.float() == 0).all()
    # dequantisation is exact: QDQ of an FP8 value is the value
    y = torch.randn(32, 64)
    d = F.qdq(y, fmt)
    assert torch.equal(F.qdq(d.float(), fmt), d)


@pytest.mark.parametrize("fmt", [F.E4M3, F.E5M2])
@pytest.mark.parametrize("bad", [float("inf"), float("-inf"), float("nan")])
def test_non_finite_input_gives_nan_everywhere(fmt, bad):
    x = torch.randn(8, 16)
    x[3, 5] = bad
    q, inv = F.quantize_ref(x, fmt)
    assert torch.isnan(q.float()).all() and torch.isnan(inv).all()
    assert (q.view(torch.uint8) == 0x7F).all()


def test_cast_writes_row_major_and_transposed_copies():
    x = torch.randn(128, 64).to(torch.bfloat16)
    slot, inv = torch.zeros(1), torch.zeros(1)
    out, out_t = torch.empty(128, 64, dtype=F.E5M2), torch.empty(64, 128, dtype=F.E5M2)
    F.quantize(x, slot, inv, F.E5M2, out=out, out_t=out_t)
    q, iv = F.quantize_ref(x, F.E5M2)
    assert torch.equal(out.view(torch.uint8), q.view(torch.uint8))
    assert torch.equal(out_t.view(torch.uint8), q.view(torch.uint8).t())
    assert float(inv) == float(iv) and float(slot) == float(x.float().abs().max())


# ------------------------------------------------------------------------------------------------ engine on the references
GQA = LlamaConfig(hidden_size=128, intermediate_size=384, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2,
                  vocab_size=512)


def _step(cfg_or_path, precision, ids):
    if isinstance(cfg_or_path, str):
        m = LlamaForCausalLM.from_pretrained(cfg_or_path, precision=precision)
    else:
        m = LlamaForCausalLM(cfg_or_path, precision=precision, seed=0)
    m.arena.grad.zero_()
    loss = float(m.forward_backward(ids, ids))
    grads = {n: p.grad.clone() for n, p in m.named_parameters()}
    return m, loss, grads


# Measured (torch 2.11 CPU, these ids): 2m golden |dloss| 4.9e-4, worst per-tensor relative gradient error 0.113
# (layers.0 q_proj); GQA tiny |dloss| 2.2e-4, worst 0.132 (layers.1 post_attention_layernorm).  e5m2 gradients keep
# 2 mantissa bits (relative rounding up to 12.5 % per element).
@pytest.mark.parametrize("model", ["golden-2m", "gqa-tiny"])
def test_fp8_mixed_matches_bf16_mixed(model):
    src = GOLDEN if model == "golden-2m" else GQA
    ids = torch.randint(0, 500, (2, 64), generator=torch.Generator().manual_seed(0))     # both vocabularies hold 500 ids
    _, l_bf, g_bf = _step(src, "bf16-mixed", ids)
    m8, l_f8, g_f8 = _step(src, "fp8-mixed", ids)
    assert m8.engine.fp8 and m8.arena.compute_dtype == torch.bfloat16
    assert abs(l_f8 - l_bf) < 2e-3
    for n, g in g_bf.items():
        err = float((g_f8[n] - g).norm() / g.norm().clamp_min(1e-12))
        assert err < 0.2, f"{n}: relative gradient error {err:.4f}"


def test_fp8_mixed_eval_forward_and_generate_run():
    m = LlamaForCausalLM.from_pretrained(GOLDEN, precision="fp8-mixed")
    m.eval()
    ids = torch.randint(0, 500, (2, 64), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        out = m(ids, labels=ids)
    assert torch.isfinite(out.loss)
    gen = m.generate(ids[:, :8], max_new_tokens=4)
    assert gen.shape == (2, 12)


# ------------------------------------------------------------------------------------------------ constructor checks
def test_cuda_shape_checks_name_the_dimension(monkeypatch):
    ok = LlamaConfig.from_pretrained("150m")
    F.check_config(ok)
    F.check_config(LlamaConfig.from_pretrained("1b"))
    F.check_config(LlamaConfig.from_pretrained("60m"))
    with pytest.raises(ValueError, match="head_dim"):
        F.check_config(LlamaConfig.from_pretrained("2m"))           # head_dim 32
    with pytest.raises(ValueError, match="intermediate_size"):
        F.check_config(LlamaConfig(hidden_size=1024, intermediate_size=2700, num_attention_heads=16))
    with pytest.raises(ValueError, match="tokens"):
        F.check_tokens(3 * 100)
    F.check_tokens(32 * 1024)
    monkeypatch.setattr(A, "_LIB", "flash")
    with pytest.raises(ValueError, match="ODB_ATTN_LIB"):
        F.check_config(ok)


def test_constructor_runs_the_checks_for_cuda_devices(monkeypatch):
    """Construction on a CUDA device consults check_config before allocating anything (mocked: no device needed)."""
    seen = []

    def fake(cfg):
        seen.append(cfg)
        raise ValueError("intermediate_size")

    monkeypatch.setattr(llama_mod.F, "check_config", fake)
    with pytest.raises(ValueError, match="intermediate_size"):
        LlamaForCausalLM(GQA, device="cuda", precision="fp8-mixed")
    assert seen == [GQA]
    LlamaForCausalLM(GQA, device="cpu", precision="fp8-mixed")       # CPU: references, no shape limits
    assert len(seen) == 1


# ------------------------------------------------------------------------------------------------ training CLI
def _free_port() -> int:
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _torchrun(nproc: int, args: list[str]) -> None:
    env = dict(os.environ, PYTHONPATH=ROOT, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="2", WANDB_MODE="disabled")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), "-m", "opendiloco_b200.train_fsdp", *args]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    if res.returncode != 0:
        pytest.fail(f"{' '.join(cmd)}\n{res.stdout[-3000:]}\n{res.stderr[-3000:]}")


def _load(path):
    with open(path, "rb") as f:
        return {d["step"]: (d["Loss"], d["lr"]) for d in pickle.load(f)}


BASE = ["--path_model", "2m", "--fake_data", "--no-torch_compile", "--lr", "1e-2", "--per_device_train_batch_size", "4",
        "--total_batch_size", "16", "--seq_length", "64", "--metric_logger_type", "dummy", "--precision", "fp8-mixed",
        "--warmup_steps", "4", "--total_steps", "100"]


@pytest.mark.parametrize("mode", ["NO_SHARD", "diloco"])
def test_train_fsdp_fp8_mixed_checkpoints_and_resumes(tmp_path, mode):
    ckpt, log1, log2 = f"{tmp_path}/ckpt", f"{tmp_path}/log1.pkl", f"{tmp_path}/log2.pkl"
    if mode == "diloco":
        extra = ["--hv.local_steps", "5", "--hv.galaxy_size", "2", "--hv.skip_load_from_peers", "--hv.fail_rank_drop",
                 "--hv.matchmaking_time", "1", "--total_batch_size", "8", "--max_steps", "12"]
        resume_at, tol = 7, 1e-2
    else:
        extra = ["--max_steps", "12", "--sharding_strategy", "NO_SHARD"]
        resume_at, tol = 8, 1e-3
    _torchrun(2, BASE + extra + ["--ckpt.path", ckpt, "--ckpt.interval", str(resume_at) if mode == "diloco" else "4",
                                 "--project", log1])
    _torchrun(2, BASE + extra + ["--ckpt.path", ckpt, "--ckpt.resume", f"{ckpt}/model_step_{resume_at}", "--project", log2])
    a, b = _load(log1), _load(log2)
    common = set(a) & set(b)
    assert common == set(range(resume_at + 1, 13))
    for s in common:
        assert abs(a[s][0] - b[s][0]) <= tol, f"loss at step {s}: {a[s][0]} vs {b[s][0]}"
    assert all(0 < a[s][0] < 20 for s in a)            # finite losses (fake data is uniform: nothing to learn)
