"""Training throughput of precision="fp8-mixed" against "bf16-mixed": the graphed micro-step (forward + LM head + backward,
CUDA-graph replay) on synthetic tokens, one GPU.  Precisions alternate, each round builds a fresh model.

    python profiles/fp8_bench.py                       # Llama-150M (32 x 1024) and Llama-1B (16 x 1024), 3 rounds
    python profiles/fp8_bench.py --profile             # separate run: share of the fp8 step per kernel class

Prints the GPU name, power limit and SM clock next to the numbers, and one JSON line per model."""
from __future__ import annotations

import argparse
import json
import re
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

from opendiloco_b200.models.config import LlamaConfig  # noqa: E402
from opendiloco_b200.models.llama import LlamaForCausalLM  # noqa: E402

SHAPES = {"150m": (32, 1024), "1b": (16, 1024)}


def gpu_info() -> str:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # pragma: no cover
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def time_steps(model, ids, steps: int, warmup: int) -> float:
    for _ in range(warmup):          # eager warm-ups, graph capture, first replay
        model.forward_backward(ids, ids, 1.0)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        model.forward_backward(ids, ids, 1.0)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def classify(name: str) -> str:
    if re.search(r"gemm_kernel<\d+, false, false, [12]>", name):      # demangled FP8 instantiations
        return "fp8 GEMM"
    if "amax_kernel" in name or "cast_kernel" in name:
        return "fp8 amax/cast"
    if "gemm_kernel" in name:
        return "bf16 GEMM (LM head)"
    if "attn" in name:
        return "attention"
    return "other"


def profile(model, ids) -> dict[str, float]:
    from torch.profiler import ProfilerActivity, profile as prof_ctx

    for _ in range(2):
        model.engine.forward_backward(ids, ids, 1.0)
    torch.cuda.synchronize()
    with prof_ctx(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            model.engine.forward_backward(ids, ids, 1.0)
        torch.cuda.synchronize()
    tot: dict[str, float] = {}
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if t > 0:
            k = classify(e.key)
            tot[k] = tot.get(k, 0.0) + t
    s = sum(tot.values())
    return {k: round(100.0 * v / s, 1) for k, v in sorted(tot.items(), key=lambda kv: -kv[1])}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="150m,1b")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--profile", action="store_true", help="kernel-class shares of the fp8 micro-step (no timing)")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "fp8_bench measures on a CUDA device"
    print("GPU:", gpu_info(), flush=True)
    for name in a.models.split(","):
        cfg = LlamaConfig.from_pretrained(name)
        B, S = SHAPES[name]
        ids = torch.randint(3, cfg.vocab_size, (B, S), device="cuda", generator=torch.Generator(device="cuda").manual_seed(0))
        if a.profile:
            m = LlamaForCausalLM(cfg, device="cuda", precision="fp8-mixed", seed=0)
            print(name, "fp8-mixed step shares (%):", json.dumps(profile(m, ids)), flush=True)
            del m
            torch.cuda.empty_cache()
            continue
        res: dict[str, list[float]] = {"bf16-mixed": [], "fp8-mixed": []}
        loss: dict[str, float] = {}
        for r in range(a.rounds):
            for prec in res:
                m = LlamaForCausalLM(cfg, device="cuda", precision=prec, seed=0)
                ms = time_steps(m, ids, a.steps, a.warmup)
                loss[prec] = float(m.engine.forward_backward(ids, ids, 1.0))
                res[prec].append(B * S / ms * 1e3)
                print(f"{name} round {r} {prec}: {ms:.1f} ms/micro-step, {res[prec][-1]:.0f} tokens/s", flush=True)
                del m
                torch.cuda.empty_cache()
        out = {"model": name, "micro_batch": [B, S], "gpu": gpu_info(),
               **{f"{p}_tokens_per_s": [round(v) for v in vs] for p, vs in res.items()},
               "speedup_median": round(sorted(res["fp8-mixed"])[len(res["fp8-mixed"]) // 2] /
                                       sorted(res["bf16-mixed"])[len(res["bf16-mixed"]) // 2], 3),
               "loss_at_init": loss}
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
