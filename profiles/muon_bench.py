"""FusedMuon on one GPU: optimizer step time against FusedAdamW and the torch baseline, Newton-Schulz GEMM throughput, and
the end-to-end cost of Muon in the training step.

    python profiles/muon_bench.py [--sizes 150m 1b] [--steps 20] [--rounds 3] [--e2e-steps 3]

1. Optimizer step (NO_SHARD, random gradients, clip 1.0, warmed up, CUDA events over ``--steps`` steps, ``--rounds``
   alternating rounds) at each size for: FusedAdamW; FusedMuon; ``torch.optim.Muon`` + ``torch.optim.AdamW(fused=True)``
   on the same parameters after ``clip_grad_norm_(foreach=True)`` (the torch baseline).
2. Newton-Schulz GEMMs: their kernel time from ``torch.profiler`` in a separate run, and TFLOP/s from the shapes
   (5 iterations of 4 m^2 n + 2 m^3 per m x n matrix, m <= n).
3. End-to-end tokens/s of the graphed micro-step at the bench shape (Llama-150M, 32 x 1024, 16 micro-batches per step)
   through ``DiLoCoTrainer.train_step``, adamw vs muon, alternating.

Prints the card name and power limit first; every number is only meaningful with them.
"""
from __future__ import annotations

import argparse
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from opendiloco_b200.models.config import LlamaConfig  # noqa: E402
from opendiloco_b200.models.llama import LlamaForCausalLM  # noqa: E402
from opendiloco_b200.optim.fused import FusedAdamW  # noqa: E402
from opendiloco_b200.optim.muon import FusedMuon, _is_muon_param  # noqa: E402


def card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


class TorchBaseline:
    def __init__(self, params):
        self.params = params
        mats = [p for p in params if _is_muon_param(p)]
        rest = [p for p in params if not _is_muon_param(p)]
        self.muon = torch.optim.Muon(mats, lr=4e-4, weight_decay=0.1, adjust_lr_fn="match_rms_adamw")
        self.adamw = torch.optim.AdamW(rest, lr=4e-4, betas=(0.9, 0.95), weight_decay=0.1, fused=True)

    def step(self):
        torch.nn.utils.clip_grad_norm_(self.params, 1.0, foreach=True)
        self.muon.step()
        self.adamw.step()


def make_opt(kind, params):
    if kind == "FusedAdamW":
        return FusedAdamW(params, lr=4e-4, betas=(0.9, 0.95), weight_decay=0.1, max_grad_norm=1.0)
    if kind == "FusedMuon":
        return FusedMuon(params, lr=4e-4, weight_decay=0.1, adjust_lr_fn="match_rms_adamw", max_grad_norm=1.0)
    return TorchBaseline(params)


def time_steps(opt, n: int) -> float:
    for _ in range(3):
        opt.step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        opt.step()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def ns_flops(params) -> float:
    tot = 0.0
    for p in params:
        if _is_muon_param(p):
            m, n = sorted(p.shape)
            tot += 5 * (4 * m * m * n + 2 * m ** 3)
    return tot


def optimizer_bench(size: str, steps: int, rounds: int) -> None:
    cfg = LlamaConfig.from_pretrained(size)
    model = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=0)
    params = list(model.parameters())
    kinds = ["FusedAdamW", "FusedMuon", "torch Muon+AdamW"]
    opts = {k: make_opt(k, params) for k in kinds}
    grad = opts["FusedAdamW"].fv.grad
    torch.manual_seed(0)
    grad.normal_().mul_(1e-3)
    for i, p in enumerate(params):                 # the torch optimizers read p.grad: views of the same flat gradient
        p.grad = opts["FusedAdamW"].fv.view_of(grad, i)
    res = {k: [] for k in kinds}
    for _ in range(rounds):
        for k in kinds:
            res[k].append(time_steps(opts[k], steps))
    flops = ns_flops(params)
    print(f"[{size}] {sum(p.numel() for p in params) / 1e6:.0f}M parameters, Newton-Schulz {flops / 1e12:.2f} TFLOP per step")
    for k in kinds:
        print(f"[{size}] optimizer step  {k:18s} " + " / ".join(f"{t:.2f}" for t in res[k]) + " ms")
    # Newton-Schulz GEMM kernel time, profiled in a run of its own
    opt = opts["FusedMuon"]
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            opt.step()
        torch.cuda.synchronize()
    ns_us = sum(e.device_time_total for e in prof.key_averages()
                if "gemm_kernel" in e.key and ("<8," in e.key or "ILi8E" in e.key)) / 3
    total_us = sum(e.device_time_total for e in prof.key_averages()) / 3
    print(f"[{size}] FusedMuon kernels {total_us / 1e3:.2f} ms per step, of which Newton-Schulz GEMMs {ns_us / 1e3:.2f} ms "
          f"= {flops / (ns_us * 1e-6) / 1e12:.0f} TFLOP/s")
    del opts, model
    torch.cuda.empty_cache()


def e2e_bench(steps: int, rounds: int) -> None:
    from opendiloco_b200.trainer import DiLoCoTrainer, TrainerConfig
    from opendiloco_b200.utils.data import SyntheticTokenLoader

    cfg = LlamaConfig.from_pretrained("150m")
    runs = {}
    for kind in ("adamw", "muon"):
        model = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=0)
        tr = DiLoCoTrainer(model, TrainerConfig(inner_optimizer=kind, grad_accum=16, local_steps=None, samples_per_step=512,
                                                warmup_steps=1000, total_steps=88_000))
        loader = SyntheticTokenLoader(32, 1024, vocab_size=cfg.vocab_size, seed=1234, with_mask=False)
        for _ in range(2):
            tr.train_step(loader)
        runs[kind] = (tr, loader, [])
    for _ in range(rounds):
        for kind, (tr, loader, out) in runs.items():
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(steps):
                tr.train_step(loader)
            b.record()
            b.synchronize()
            out.append(512 * 1024 * steps / (a.elapsed_time(b) / 1e3))
    for kind, (_, _, out) in runs.items():
        print(f"[150m e2e] {kind:6s} " + " / ".join(f"{t / 1e3:.1f}k" for t in out) + " tokens/s")
    ra = sum(runs["adamw"][2]) / rounds
    rm = sum(runs["muon"][2]) / rounds
    print(f"[150m e2e] muon costs {100 * (1 - rm / ra):.2f} % of adamw's tokens/s (mean of {rounds} rounds)")


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", nargs="+", default=["150m", "1b"])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--e2e-steps", type=int, default=3)
    ap.add_argument("--no-e2e", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("muon_bench.py measures the GPU: no CUDA device found")
    print(f"card: {card()}")
    for size in a.sizes:
        optimizer_bench(size, a.steps, a.rounds)
    if not a.no_e2e:
        e2e_bench(a.e2e_steps, a.rounds)


if __name__ == "__main__":
    main()
