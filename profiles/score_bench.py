"""Scoring throughput on the H100: ``model.score`` against ``model(ids).logits`` + log_softmax + gather and against
transformers' forward + log_softmax + gather (bf16, same weights, same GPU, one process), plus a per-kernel split of one
``score`` call into the layer program and the LM head (kLCEScore GEMM + lce_score_finalize).

    python profiles/score_bench.py                          # presets 150m, 1b x B x S in {8x1024, 32x1024, 16x2048}
    python profiles/score_bench.py --presets 150m --shapes 8x1024 --no-hf

Weights are random from a seed.  Every timing uses CUDA events around work repeated for at least --window seconds after a
warm-up; tokens/s counts the B x S input tokens of a call.  The three arms are timed in turn for each shape.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch  # noqa: E402

from generate_bench import card, hf_model, timed  # noqa: E402
from opendiloco_b200.models.config import LlamaConfig  # noqa: E402
from opendiloco_b200.models.llama import LlamaForCausalLM  # noqa: E402


def _gather_logprobs(logits: torch.Tensor, ids: torch.Tensor) -> torch.Tensor:
    return torch.log_softmax(logits[:, :-1].float(), dim=-1).gather(2, ids[:, 1:, None])[..., 0]


def kernel_split(model, ids) -> dict:
    """GPU time of one score call by kernel: the LM head (scoring GEMM + finalize) against everything else."""
    from torch.profiler import ProfilerActivity, profile

    model.score(ids)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.score(ids)
        torch.cuda.synchronize()
    head = layers = 0.0
    for e in prof.key_averages():
        if e.device_type != torch.autograd.DeviceType.CUDA or e.key.startswith(("Memcpy", "Memset")):
            continue
        us = e.self_device_time_total
        if "gemm_kernel<7," in e.key or "lce_score_finalize" in e.key:
            head += us
        else:
            layers += us
    return {"layers_ms": round(layers / 1e3, 3), "lm_head_ms": round(head / 1e3, 3),
            "lm_head_share": round(head / max(head + layers, 1e-9), 3)}


def bench(name: str, shapes, window: float, with_hf: bool) -> None:
    cfg = LlamaConfig.from_pretrained(name)
    model = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=0).eval()
    hf = hf_model(model) if with_hf else None
    for B, S in shapes:
        ids = torch.randint(0, cfg.vocab_size, (B, S), generator=torch.Generator().manual_seed(B * 7 + S)).cuda()
        row = {"preset": name, "B": B, "S": S}
        lp = model.score(ids).logprobs
        t = timed(lambda: model.score(ids), window)
        row["score_tokens_per_s"] = round(B * S / t, 1)
        row.update(kernel_split(model, ids))
        model.engine.score_state = None

        def via_logits():
            with torch.no_grad():
                return _gather_logprobs(model(ids).logits, ids)

        ref = via_logits()
        row["max_abs_diff_vs_logits_path"] = round((lp[:, 1:] - ref).abs().max().item(), 5)
        del ref
        t = timed(via_logits, window)
        row["logits_path_tokens_per_s"] = round(B * S / t, 1)
        model.engine._ws.clear()
        model.engine._graphs.clear()
        torch.cuda.empty_cache()
        if hf is not None:
            def via_hf():
                with torch.no_grad():
                    return _gather_logprobs(hf(ids).logits, ids)

            t = timed(via_hf, window)
            row["hf_tokens_per_s"] = round(B * S / t, 1)
            torch.cuda.empty_cache()
        row["speedup_vs_logits_path"] = round(row["score_tokens_per_s"] / row["logits_path_tokens_per_s"], 2)
        if hf is not None:
            row["speedup_vs_hf"] = round(row["score_tokens_per_s"] / row["hf_tokens_per_s"], 2)
        print(json.dumps(row), flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--presets", default="150m,1b")
    ap.add_argument("--shapes", default="8x1024,32x1024,16x2048", help="comma-separated BxS")
    ap.add_argument("--window", type=float, default=1.0, help="seconds of timed work per number")
    ap.add_argument("--no-hf", action="store_true", help="skip the transformers comparison")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "score_bench needs a GPU"
    print(json.dumps(card()), flush=True)
    shapes = [tuple(int(v) for v in s.split("x")) for s in a.shapes.split(",")]
    for name in a.presets.split(","):
        bench(name, shapes, a.window, not a.no_hf)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
