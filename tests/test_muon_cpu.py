"""FusedMuon on CPU (the PyTorch reference path of every Muon kernel): agreement with torch.optim.Muon + torch.optim.AdamW,
GradScaler skips, state_dict round trip and argument errors."""
import copy
import json
import os
import pickle
import socket
import subprocess
import sys

import pytest
import torch

from opendiloco_b200.ops import muon as M
from opendiloco_b200.optim.fused import clip_grad_norm_
from opendiloco_b200.optim.muon import FusedMuon


def _models():
    torch.manual_seed(0)
    a = torch.nn.Sequential(torch.nn.Linear(64, 256), torch.nn.LayerNorm(256), torch.nn.Linear(256, 128),
                            torch.nn.Linear(128, 512, bias=False))
    return a, copy.deepcopy(a)


def _torch_pair(model, lr, wd, momentum, nesterov, adjust):
    mats = [p for p in model.parameters() if p.ndim == 2]
    rest = [p for p in model.parameters() if p.ndim != 2]
    return (torch.optim.Muon(mats, lr=lr, weight_decay=wd, momentum=momentum, nesterov=nesterov, adjust_lr_fn=adjust),
            torch.optim.AdamW(rest, lr=lr, betas=(0.9, 0.95), eps=1e-8, weight_decay=wd))


@pytest.mark.parametrize("adjust,nesterov", [(None, True), ("original", True), ("match_rms_adamw", True), (None, False)])
def test_matches_torch_muon_and_adamw(adjust, nesterov):
    ours, ref = _models()
    lr, wd = 2e-2, 0.1
    opt = FusedMuon(ours.parameters(), lr=lr, weight_decay=wd, nesterov=nesterov, adjust_lr_fn=adjust, max_grad_norm=1.0)
    tmuon, tadam = _torch_pair(ref, lr, wd, 0.95, nesterov, adjust)
    g = torch.Generator().manual_seed(1)
    for step in range(3):
        before = [q.detach().clone() for q in ref.parameters()]
        for p, q in zip(ours.parameters(), ref.parameters()):
            gr = torch.randn(p.shape, generator=g) * 0.3
            p.grad.copy_(gr)
            q.grad = gr.clone()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), 1.0)
        tmuon.step()
        tadam.step()
        opt.step()
        for p, q, b in zip(ours.parameters(), ref.parameters(), before):
            if p.ndim == 2:
                du, dt = p.detach() - b, q.detach() - b
                rel = float((du - dt).norm() / dt.norm())
                assert rel < 3e-2, (step, p.shape, rel)
                p.data.copy_(q.detach())      # keep both runs on the same weights: compare one update at a time
            else:
                assert torch.allclose(p, q, atol=2e-6), (step, (p - q).abs().max())


def test_clip_handoff_and_groups():
    ours, _ = _models()
    opt = FusedMuon(ours.parameters(), lr=1e-2, adamw_lr=3e-3)
    assert [len(g["params"]) for g in opt.param_groups] == [3, 4]   # 3 matrices | 2 biases + LayerNorm weight and bias
    assert opt.param_groups[1]["lr"] == 3e-3
    for p in ours.parameters():
        p.grad.fill_(1.0)
    n = clip_grad_norm_(ours, 1.0, optimizer=opt)          # deferred into the step, as for FusedAdamW
    total = sum(p.numel() for p in ours.parameters())
    assert abs(float(n) - total ** 0.5) < 1e-3 * total ** 0.5
    opt.step()
    assert abs(float(opt.stats[1]) - 1.0 / total ** 0.5) < 1e-6


def test_overflow_skips_the_step_exactly():
    ours, _ = _models()
    opt = FusedMuon(ours.parameters(), lr=1e-2, max_grad_norm=1.0)
    for p in ours.parameters():
        p.grad.normal_()
    opt.step()
    snap = [t.clone() for t in (opt.fv.flat, opt.exp_avg, opt.exp_avg_sq)]
    for p in ours.parameters():
        p.grad.normal_()
    next(ours.parameters()).grad[0, 0] = float("inf")
    opt.step(_check_inf=True)
    assert int(opt._flag.item()) == 1
    for a, b in zip(snap, (opt.fv.flat, opt.exp_avg, opt.exp_avg_sq)):
        assert torch.equal(a, b)


def test_state_dict_round_trip():
    a, b = _models()
    oa = FusedMuon(a.parameters(), lr=1e-2)
    g = [torch.randn(p.shape) for p in a.parameters()]
    for p, gr in zip(a.parameters(), g):
        p.grad.copy_(gr)
    oa.step()
    sd = copy.deepcopy(oa.state_dict())
    assert set(sd["state"][0]) == {"momentum_buffer"}
    assert {"step", "exp_avg", "exp_avg_sq"} <= set(sd["state"][len(sd["param_groups"][0]["params"])])
    b.load_state_dict(a.state_dict())
    ob = FusedMuon(b.parameters(), lr=1e-2)
    ob.load_state_dict(sd)
    for o, m in ((oa, a), (ob, b)):
        for p, gr in zip(m.parameters(), g):
            p.grad.copy_(gr)
        o.step()
    for p, q in zip(a.parameters(), b.parameters()):
        assert torch.equal(p, q)


def test_batched_gemm_reference_rounds_once():
    torch.manual_seed(0)
    a = torch.randn(2, 64, 128).to(torch.bfloat16)
    d = torch.randn(2, 64, 64).to(torch.bfloat16)
    c = torch.empty(2, 64, 64, dtype=torch.bfloat16)
    M.gemm_batched_axpby(a, a, c, d, 0.5, -2.0, b_mn=False)
    want = (0.5 * (a.float() @ a.float().transpose(1, 2)) - 2.0 * d.float()).to(torch.bfloat16)
    assert torch.equal(c, want)


def test_argument_errors():
    ours, _ = _models()
    with pytest.raises(ValueError):
        FusedMuon(ours.parameters(), shard=True)
    with pytest.raises(ValueError):
        FusedMuon(ours.parameters(), adjust_lr_fn="bogus")


# ------------------------------------------------------------------------------------------------ arena-backed golden model
def test_golden_model_selection_and_agreement_with_torch(ref_model_dir):
    from opendiloco_b200.models.llama import LlamaForCausalLM

    model = LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")
    params = list(model.parameters())
    names = [p._odb_name for p in params]
    ref = [p.detach().clone().requires_grad_(True) for p in params]
    opt = FusedMuon(params, lr=2e-2, weight_decay=0.1, max_grad_norm=1.0, adjust_lr_fn="match_rms_adamw")
    muon_names = {names[i] for i in opt._muon_idx}
    want = {n for n in names if any(f".{k}." in n for k in ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj",
                                                            "down_proj"))}
    assert muon_names == want and len(want) == 7 * model.config.num_hidden_layers
    assert "model.embed_tokens.weight" not in muon_names and "lm_head.weight" not in muon_names
    is_m = [n in want for n in names]
    tmuon = torch.optim.Muon([q for q, m in zip(ref, is_m) if m], lr=2e-2, weight_decay=0.1, adjust_lr_fn="match_rms_adamw")
    tadam = torch.optim.AdamW([q for q, m in zip(ref, is_m) if not m], lr=2e-2, betas=(0.9, 0.95), weight_decay=0.1)
    g = torch.Generator().manual_seed(3)
    for step in range(3):
        before = [q.detach().clone() for q in ref]
        for p, q in zip(params, ref):
            gr = torch.randn(p.shape, generator=g) * 0.1
            p.grad.copy_(gr)
            q.grad = gr.clone()
        torch.nn.utils.clip_grad_norm_(ref, 1.0)
        tmuon.step()
        tadam.step()
        opt.step()
        for p, q, b, m in zip(params, ref, before, is_m):
            if m:
                rel = float(((p.detach() - b) - (q.detach() - b)).norm() / (q.detach() - b).norm())
                assert rel < 3e-2, (step, p._odb_name, rel)
                p.data.copy_(q.detach())
            else:
                assert torch.allclose(p, q, atol=2e-6), (step, p._odb_name)


# ------------------------------------------------------------------------------------------------ checkpoints
def _tiny_run(kind, tmp, name):
    from opendiloco_b200.models.llama import LlamaForCausalLM
    from opendiloco_b200.optim.fused import FusedAdamW
    from opendiloco_b200.utils.training import get_cosine_schedule_with_warmup

    model = LlamaForCausalLM.from_pretrained("2m", precision="32-true", seed=0)
    opt = FusedMuon(model.parameters(), lr=1e-2, adamw_lr=3e-3) if kind == "muon" else FusedAdamW(model.parameters(), lr=1e-2)
    sched = get_cosine_schedule_with_warmup(opt, num_warmup_steps=2, num_training_steps=10)
    return model, opt, sched, f"{tmp}/{name}"


@pytest.mark.parametrize("saved,resumed", [("muon", "adamw"), ("adamw", "muon"), ("muon", "muon")])
def test_checkpoint_tag_and_cross_optimizer_resume(tmp_path, saved, resumed):
    from opendiloco_b200.utils.ckpt import load_checkpoint, save_checkpoint

    model, opt, sched, path = _tiny_run(saved, tmp_path, "ck")
    for _ in range(3):
        opt.fv.grad.normal_()
        opt.step()
        sched.step()
    save_checkpoint(path, model, opt, scheduler=sched, rank=0)
    meta = json.load(open(f"{path}/.metadata"))
    assert meta.get("inner_optimizer") == ("muon" if saved == "muon" else None)
    model2, opt2, sched2, _ = _tiny_run(resumed, tmp_path, "unused")
    if saved != resumed:
        with pytest.raises(ValueError, match="inner optimizer"):
            load_checkpoint(path, model2, opt2, scheduler=sched2, rank=0)
        return
    load_checkpoint(path, model2, opt2, scheduler=sched2, rank=0)
    assert torch.equal(opt2.exp_avg, opt.exp_avg) and torch.equal(opt2.fv.flat, opt.fv.flat)
    assert [g["lr"] for g in opt2.param_groups] == [g["lr"] for g in opt.param_groups]   # both groups' lr restored
    assert opt2.param_groups[0]["lr"] != opt2.param_groups[1]["lr"]


def test_converter_refuses_muon_checkpoints(tmp_path):
    from opendiloco_b200.utils.ckpt import save_checkpoint
    from opendiloco_b200.utils.dcp_interop import export_dcp

    model, opt, sched, path = _tiny_run("muon", tmp_path, "ck")
    save_checkpoint(path, model, opt, scheduler=sched, rank=0)
    with pytest.raises(ValueError, match="only AdamW"):
        export_dcp(path, f"{tmp_path}/dcp")


# ------------------------------------------------------------------------------------------------ training entry points
def test_sharded_strategies_are_rejected_before_any_work():
    from opendiloco_b200.models.llama import LlamaForCausalLM
    from opendiloco_b200.train_fsdp import Config, train
    from opendiloco_b200.trainer import DiLoCoTrainer, TrainerConfig

    with pytest.raises(ValueError, match="NO_SHARD"):
        train(Config(path_model="2m", fake_data=True, inner_optimizer="muon", sharding_strategy="SHARD_GRAD_OP",
                     metric_logger_type="dummy"))
    model = LlamaForCausalLM.from_pretrained("2m", precision="32-true")
    with pytest.raises(ValueError, match="NO_SHARD"):
        DiLoCoTrainer(model, TrainerConfig(inner_optimizer="muon", sharding_strategy="FULL_SHARD", local_steps=None))


def _free_port() -> int:
    with socket.socket(socket.AF_INET, socket.SOCK_STREAM) as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _torchrun(nproc: int, args: list[str]) -> None:
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=root, CUDA_VISIBLE_DEVICES="", OMP_NUM_THREADS="2", WANDB_MODE="disabled")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), "-m", "opendiloco_b200.train_fsdp", *args]
    res = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    if res.returncode != 0:
        pytest.fail(f"{' '.join(cmd)}\n{res.stdout[-3000:]}\n{res.stderr[-3000:]}")


def _losses(path):
    with open(path, "rb") as f:
        return {d["step"]: d["Loss"] for d in pickle.load(f)}


BASE = ["--path_model", "2m", "--fake_data", "--no-torch_compile", "--lr", "1e-2", "--per_device_train_batch_size", "4",
        "--total_batch_size", "16", "--seq_length", "64", "--metric_logger_type", "dummy", "--inner-optimizer", "muon",
        "--muon-momentum", "0.9", "--warmup_steps", "4", "--total_steps", "100"]


@pytest.mark.parametrize("mode", ["NO_SHARD", "diloco"])
def test_train_fsdp_muon_checkpoints_and_resumes(tmp_path, mode):
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
    sub = "/diloco_rank_0" if mode == "diloco" else ""
    assert json.load(open(f"{ckpt}/model_step_{resume_at}{sub}/.metadata"))["inner_optimizer"] == "muon"
    _torchrun(2, BASE + extra + ["--ckpt.path", ckpt, "--ckpt.resume", f"{ckpt}/model_step_{resume_at}", "--project", log2])
    a, b = _losses(log1), _losses(log2)
    common = set(a) & set(b)
    assert common == set(range(resume_at + 1, 13))
    for s in common:
        assert abs(a[s] - b[s]) <= tol, f"loss at step {s}: {a[s]} vs {b[s]}"
    assert all(0 < a[s] < 20 for s in a)
