"""FusedMuon kernels on the H100: batched axpby GEMMs against fp32 torch, Newton-Schulz against fp64, a full step on an
arena-backed Llama against the PyTorch reference path on the same GPU, determinism and kernel ownership."""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from opendiloco_b200.ops import kernels as K
from opendiloco_b200.ops import muon as M
from opendiloco_b200.optim.muon import FusedMuon, adjust_lr_ratio

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
COEFFS = (3.4445, -4.775, 2.0315)


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


@pytest.mark.parametrize("b_mn,batch,m,n,k", [(False, 3, 1024, 1024, 2688), (False, 2, 256, 256, 2048),
                                              (True, 3, 1024, 2688, 1024), (True, 2, 2048, 5632, 2048)])
def test_batched_axpby_gemm(b_mn, batch, m, n, k):
    g = torch.Generator(device=DEV).manual_seed(0)
    a = torch.randn(batch, m, k, device=DEV, generator=g).to(torch.bfloat16)
    b = torch.randn((batch, k, n) if b_mn else (batch, n, k), device=DEV, generator=g).to(torch.bfloat16)
    d = torch.randn(batch, m, n, device=DEV, generator=g).to(torch.bfloat16)
    c = torch.empty(batch, m, n, device=DEV, dtype=torch.bfloat16)
    M.gemm_batched_axpby(a, b, c, d, 0.5, -1.5, b_mn)
    ref = 0.5 * torch.bmm(a.float(), b.float() if b_mn else b.float().transpose(1, 2)) - 1.5 * d.float()
    assert _rel(c, ref) < 4e-3
    for i in range(batch):                      # one batched call == per-matrix calls, bit for bit
        ci = torch.empty(1, m, n, device=DEV, dtype=torch.bfloat16)
        M.gemm_batched_axpby(a[i:i + 1].contiguous(), b[i:i + 1].contiguous(), ci, d[i:i + 1].contiguous(), 0.5, -1.5, b_mn)
        assert torch.equal(ci[0], c[i])
    c0 = torch.empty_like(c)
    M.gemm_batched_axpby(a, b, c0, None, 1.0, 0.0, b_mn)
    assert _rel(c0, torch.bmm(a.float(), b.float() if b_mn else b.float().transpose(1, 2))) < 4e-3


def _ns64(x):
    a, b, c = COEFFS
    for _ in range(5):
        A = x @ x.T
        x = a * x + (b * A + c * A @ A) @ x
    return x


@pytest.mark.parametrize("rows,cols", [(1024, 1024), (2688, 1024), (1024, 2688), (256, 2048), (2048, 2048), (5632, 2048)])
def test_newton_schulz_against_fp64(rows, cols):
    from torch.optim._muon import _zeropower_via_newtonschulz

    g = torch.randn(rows, cols, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    u = g.T if rows > cols else g
    m, n = u.shape
    want = _ns64((u / u.norm()).double())
    x = (u / u.norm()).to(torch.bfloat16).contiguous().view(1, m, n)
    bufs = [torch.empty(1, m, n, device=DEV, dtype=torch.bfloat16)] + [torch.empty(1, m, m, device=DEV, dtype=torch.bfloat16)
                                                                        for _ in range(2)]
    ours = M.newton_schulz(x, COEFFS, 5, *bufs)[0]
    theirs = _zeropower_via_newtonschulz(g, COEFFS, 5, 1e-7)
    theirs = theirs.T if rows > cols else theirs
    e_ours, e_torch = _rel(ours, want), _rel(theirs, want)
    print(f"NS {rows}x{cols}: ours {e_ours:.3e} torch bf16 {e_torch:.3e}")
    assert e_ours <= 1.25 * e_torch


def _llama():
    from opendiloco_b200.models.config import LlamaConfig
    from opendiloco_b200.models.llama import LlamaForCausalLM

    cfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=2, num_attention_heads=16,
                      num_key_value_heads=4, vocab_size=4096)
    return LlamaForCausalLM(cfg, device=DEV, precision="bf16-mixed", seed=0)


def _step(model, theta, grad):
    opt = FusedMuon(model.parameters(), lr=2e-2, weight_decay=0.1, max_grad_norm=1.0, adjust_lr_fn="match_rms_adamw")
    opt.fv.flat.copy_(theta)
    opt.fv.grad.copy_(grad)
    opt.step()
    torch.cuda.synchronize()
    return opt


def test_full_step_matches_reference_and_is_deterministic():
    model = _llama()
    fv0 = FusedMuon(model.parameters()).fv
    theta = fv0.flat.clone()
    grad = torch.randn(fv0.grad.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(2)) * 1e-3
    opt = _step(model, theta, grad)
    fv = opt.fv
    assert not opt._ref_idx and len(opt._muon_idx) == 14
    hp = opt._hp.cpu()
    part = grad.cpu().double().pow(2).sum().float().reshape(1)      # the whole flat gradient, as the norm pass sees it
    coef = M.clip_coef_ref(hp, part, 1)
    mg = opt.param_groups[0]
    worst = 0.0
    for i in opt._muon_idx:
        p = fv.params[i]
        t = fv.view_of(theta, i).clone()
        M.muon_update_ref(t, fv.view_of(grad, i), torch.zeros_like(t), None, coef, mg["lr"], mg["weight_decay"], mg["momentum"],
                          True, COEFFS, 5, 1e-7, adjust_lr_ratio("match_rms_adamw", p.shape), False)
        base = fv.view_of(theta, i)
        rel = _rel(fv.view_of(fv.flat, i) - base, t - base)
        worst = max(worst, rel)
        assert torch.equal(fv.shadow[fv.offsets[i]:fv.offsets[i] + p.numel()], fv.view_of(fv.flat, i).reshape(-1).to(torch.bfloat16))
    print(f"kernel vs reference update, worst relative error: {worst:.3e}")
    # measured on an H100 80GB HBM3 (400 W): 6.3e-3 (GEMM accumulation order vs cuBLAS fp32 products); bound = 1.5x that
    assert worst < 9.5e-3
    for i in opt._adamw_idx:
        sl = slice(fv.offsets[i], fv.offsets[i] + fv.params[i].numel())
        t = theta[sl].cpu().clone()
        K.adamw_step(t, grad[sl].cpu().clone(), torch.zeros_like(t), torch.zeros_like(t), None, hp, part, 1, None, None)
        assert torch.allclose(fv.flat[sl].cpu(), t, rtol=0, atol=2e-6)
    # the same step again from the same state (the arena's master buffer is reused): bit-identical master weights
    first = int(K.checksum_i32(fv.flat))
    again = _step(model, theta, grad)
    assert int(K.checksum_i32(again.fv.flat)) == first


def test_step_launches_no_library_kernel():
    _in_fresh_process("_step_launches_no_library_kernel")


def _step_launches_no_library_kernel():
    model = _llama()
    opt = FusedMuon(model.parameters(), lr=1e-2, max_grad_norm=1.0)
    opt.fv.grad.normal_()
    opt.step()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        opt.fv.grad.normal_()
        torch.cuda.synchronize()
        opt.step()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
    lib = [n for n in names if any(s in n.lower() for s in ("cublas", "cutlass", "xmma", "nvjet", "gemv", "cudnn"))]
    assert not lib, lib
    assert any("gemm_kernel" in n for n in names) and any("muon_apply" in n for n in names), names


def test_graphed_micro_step_survives_optimizer_steps():
    from opendiloco_b200.trainer import DiLoCoTrainer, TrainerConfig
    from opendiloco_b200.utils.data import SyntheticTokenLoader

    model = _llama()
    tr = DiLoCoTrainer(model, TrainerConfig(inner_optimizer="muon", grad_accum=2, local_steps=None, samples_per_step=4,
                                            warmup_steps=2, total_steps=10))
    loader = SyntheticTokenLoader(2, 256, vocab_size=model.config.vocab_size, seed=0, with_mask=False)
    # the micro-step is captured on its third call (second step); the NS scratch is allocated by the first optimizer step
    losses = [float(tr.train_step(loader).item()) for _ in range(2)]
    version, graphs = model.arena.version, dict(model.engine._graphs)
    assert graphs and all(st["graph"] is not None for st in graphs.values())
    losses += [float(tr.train_step(loader).item()) for _ in range(3)]
    assert model.arena.version == version
    assert all(model.engine._graphs[k] is st and st["graph"] is g["graph"] for k, st, g in
               ((k, model.engine._graphs[k], graphs[k]) for k in graphs))
    assert all(0 < x < 20 for x in losses), losses


def _bigram_stream(steps, B, S, V, seed):
    """Each token follows a fixed successor table with probability 0.85, else a uniform draw from 512 ids."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    vocab = torch.randperm(V, device="cuda", generator=g)[:512]
    succ = torch.randint(0, 512, (512,), device="cuda", generator=g)
    out = []
    for _ in range(steps):
        idx = torch.empty(B, S, dtype=torch.long, device="cuda")
        idx[:, 0] = torch.randint(0, 512, (B,), device="cuda", generator=g)
        noise = torch.randint(0, 512, (B, S), device="cuda", generator=g)
        keep = torch.rand(B, S, device="cuda", generator=g) < 0.85
        for s in range(1, S):
            idx[:, s] = torch.where(keep[:, s], succ[idx[:, s - 1]], noise[:, s])
        out.append(vocab[idx])
    return out


def _train(kind, batches, cfg):
    from opendiloco_b200.models.llama import LlamaForCausalLM
    from opendiloco_b200.optim.fused import FusedAdamW

    m = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=0)
    if kind == "muon":
        opt = FusedMuon(m.parameters(), lr=1e-3, weight_decay=0.0, adjust_lr_fn="match_rms_adamw", max_grad_norm=1.0)
    else:
        opt = FusedAdamW(m.parameters(), lr=1e-3, betas=(0.9, 0.95), weight_decay=0.0, max_grad_norm=1.0)
    losses = []
    for ids in batches:
        opt.zero_grad()
        losses.append(m.forward_backward(ids, ids, 1.0).item())
        opt.step()                      # writes the bf16 compute weights too
    return losses


def test_muon_training_learns_the_bigram_stream():
    from opendiloco_b200.models.config import LlamaConfig

    cfg = LlamaConfig.from_pretrained("60m")
    batches = _bigram_stream(200, 8, 256, cfg.vocab_size, seed=0)
    lm, la = _train("muon", batches, cfg), _train("adamw", batches, cfg)
    tail_m, tail_a = sum(lm[-20:]) / 20, sum(la[-20:]) / 20
    print(f"first loss {lm[0]:.4f}; last-20 mean: muon {tail_m:.4f}, adamw {tail_a:.4f}")
    assert tail_m < 0.5 * lm[0], "the stream was not learned"


def _replica_worker(rank, world, port, out):
    import torch.distributed as dist

    from opendiloco_b200.models.config import LlamaConfig
    from opendiloco_b200.models.llama import LlamaForCausalLM

    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        cfg = LlamaConfig(hidden_size=512, intermediate_size=1408, num_hidden_layers=2, num_attention_heads=8,
                          num_key_value_heads=4, vocab_size=2048)
        model = LlamaForCausalLM(cfg, device=torch.device("cuda", rank), precision="bf16-mixed", seed=0)
        opt = FusedMuon(model.parameters(), lr=1e-2, max_grad_norm=1.0, dp_group=dist.group.WORLD)
        g = torch.Generator(device="cuda").manual_seed(100 + rank)          # every rank sees different gradients
        for _ in range(3):
            opt.fv.grad.normal_(generator=g)
            opt.step()
            opt.zero_grad()
        sums = [torch.zeros(1, dtype=torch.int64, device="cuda") for _ in range(world)]
        dist.all_gather(sums, K.checksum_i32(opt.fv.flat))
        if rank == 0:
            torch.save([int(x) for x in sums], out)
    finally:
        dist.destroy_process_group()


def test_no_shard_replicas_stay_bit_identical(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    import socket

    import torch.multiprocessing as mp

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    out = os.path.join(tmp_path, "sums.pt")
    mp.spawn(_replica_worker, args=(2, port, out), nprocs=2, join=True)
    sums = torch.load(out)
    assert len(set(sums)) == 1, sums


def _in_fresh_process(fn: str) -> None:
    """Run ``fn`` of this module in a new Python process and fail with its traceback if it fails.  Used by the tests that
    read kernel names from the CUDA profiler: late in a long pytest process the profiler intermittently records no GPU
    activity at all, while a fresh process records every launch."""
    here = Path(__file__).resolve()
    code = f"import sys; sys.path[:0] = [{str(here.parents[1])!r}, {str(here.parent)!r}]; import {here.stem}; {here.stem}.{fn}()"
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=here.parents[1], timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-6000:]
