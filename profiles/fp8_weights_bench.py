"""FP8 weight-only generation on the H100: ``generate(fp8_weights=True)`` against bf16 ``generate``.

    python profiles/fp8_weights_bench.py                      # every part, one JSON line per measurement
    python profiles/fp8_weights_bench.py --parts kernels --models 1b

Parts:

1. ``decode``: 150m and 1b presets (random weights), B in {1, 8, 64}, prompts of 128 and 1024 random tokens, 256 new
   tokens, greedy, no EOS.  Decode ms/token = (time of a 256-token call - time of a 1-token call) / 255, so prefill is
   left out.  bf16 and fp8 run on two model objects with the same weights (each keeps its own caches and decode graph)
   and are alternated call by call, --reps times; the minimum is reported.
2. ``kernels``: every projection of each preset at M in {1, 8, 64}: the skinny e4m3 GEMM and the bf16 GEMM on Ŵ (CUDA
   events around one CUDA graph of 200 back-to-back launches), with the bytes each must read computed from the shapes (weights, row factors,
   x, y) and the rate as a share of the 3.35 TB/s HBM3 data-sheet figure.  Also the quantisation of all projections
   (one launch) per call.
3. ``quality``: a 60m preset trained here on sequences that repeat a random span (``lookup_bench.py``'s copy task; random
   weights say nothing about quality): held-out perplexity with and without FP8 weights, and greedy agreement.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from generate_bench import card  # noqa: E402
from opendiloco_b200.models import fp8_weights as W8  # noqa: E402
from opendiloco_b200.models.config import LlamaConfig  # noqa: E402
from opendiloco_b200.models.llama import LlamaForCausalLM  # noqa: E402
from opendiloco_b200.ops import fp8w as FW  # noqa: E402
from opendiloco_b200.ops import gemm as G  # noqa: E402

HBM = 3.35e12


def timed_call(fn) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def event_time(fn, n: int) -> float:
    """Seconds per call: n back-to-back calls captured in one CUDA graph (so host launch cost is not timed), replayed
    after a warm-up replay."""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n):
            fn()
    g.replay()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    g.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / 1e3 / n


def decode(models: list[str], batches: list[int], prompts: list[int], new: int, reps: int) -> None:
    for name in models:
        bf = LlamaForCausalLM(LlamaConfig.from_pretrained(name), device="cuda", precision="bf16-mixed", seed=0).eval()
        f8 = LlamaForCausalLM(LlamaConfig.from_pretrained(name), device="cuda", precision="bf16-mixed", seed=0).eval()
        for B in batches:
            for P in prompts:
                ids = torch.randint(3, bf.config.vocab_size, (B, P), generator=torch.Generator().manual_seed(B + P)).cuda()
                calls = {"bf16": lambda n: bf.generate(ids, max_new_tokens=n, eos_token_id=[]),
                         "fp8": lambda n: f8.generate(ids, max_new_tokens=n, eos_token_id=[], fp8_weights=True)}
                best = {(m, n): math.inf for m in calls for n in (1, new)}
                for m in calls:                        # warm-up: caches and decode graphs of this shape
                    calls[m](new)
                for _ in range(reps):
                    for n in (new, 1):
                        for m in calls:
                            best[m, n] = min(best[m, n], timed_call(lambda: calls[m](n)))
                ms = {m: (best[m, new] - best[m, 1]) / (new - 1) * 1e3 for m in calls}
                agree = float((calls["bf16"](new)[:, P:] == calls["fp8"](new)[:, P:]).float().mean())
                print(json.dumps({"part": "decode", "model": name, "B": B, "prompt": P, "new_tokens": new,
                                  "bf16_ms_per_token": round(ms["bf16"], 4), "fp8_ms_per_token": round(ms["fp8"], 4),
                                  "bf16_tokens_per_s": round(B / ms["bf16"] * 1e3, 1), "fp8_tokens_per_s": round(B / ms["fp8"] * 1e3, 1),
                                  "speedup": round(ms["bf16"] / ms["fp8"], 3), "greedy_tokens_equal_bf16": round(agree, 4),
                                  "reps": reps}), flush=True)
        del bf, f8
        torch.cuda.empty_cache()


def kernels(models: list[str], ms: list[int]) -> None:
    for name in models:
        cfg = LlamaConfig.from_pretrained(name)
        cfg.num_hidden_layers = min(cfg.num_hidden_layers, 2)
        model = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=0)
        fw = W8.fp8_weights(model)
        full = LlamaConfig.from_pretrained(name).num_hidden_layers
        t = event_time(lambda: fw.refresh(model.arena), 20)
        nbytes = sum(w.numel() for k in W8.KINDS for w in [W8.arena_weight(model.arena, k, 0)]) * cfg.num_hidden_layers
        print(json.dumps({"part": "quantise", "model": name, "layers": cfg.num_hidden_layers, "us": round(t * 1e6, 1),
                          "us_per_call_all_layers": round(t * 1e6 * full / cfg.num_hidden_layers, 1),
                          "TB_per_s": round(nbytes * (2 + 1 + 2) / t / 1e12, 3)}), flush=True)
        for kind in W8.KINDS:
            N, K = W8.arena_weight(model.arena, kind, 0).shape
            for M in ms:
                x = torch.randn(M, K, device="cuda").to(torch.bfloat16)
                out = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
                act = torch.empty(M, N // 2, dtype=torch.bfloat16, device="cuda") if kind == "gu" else None
                t8 = event_time(lambda: fw.linear(kind, 0, x, out, act=act), 200)
                t16 = event_time(lambda: G.mm_nt(x, fw.weight(kind, 0), out=out), 200)
                io = M * K * 2 + M * N * 2 + (M * N // 2 * 2 if act is not None else 0)
                b8, b16 = N * K + N * 4 + io, N * K * 2 + io
                print(json.dumps({"part": "kernels", "model": name, "proj": kind, "M": M, "N": N, "K": K, "splits": fw.splits[kind],
                                  "fp8_us": round(t8 * 1e6, 2), "bf16_us": round(t16 * 1e6, 2),
                                  "fp8_TB_per_s": round(b8 / t8 / 1e12, 3), "fp8_share_of_hbm": round(b8 / t8 / HBM, 3),
                                  "bf16_TB_per_s": round(b16 / t16 / 1e12, 3), "bf16_share_of_hbm": round(b16 / t16 / HBM, 3)}),
                      flush=True)
        del model, fw
        torch.cuda.empty_cache()


def quality(steps: int) -> None:
    from lookup_bench import CUE, SPAN, copy_batch, train_copy_model

    model = train_copy_model(steps, 32, seed=0)
    g = torch.Generator().manual_seed(777)
    nll = {False: 0.0, True: 0.0}
    n_tok = 0
    for _ in range(8):
        ids = copy_batch(16, g).cuda()
        for f in nll:
            nll[f] -= float(model.score(ids, fp8_weights=f).logprobs[:, 1:].double().sum())
        n_tok += ids.shape[0] * (ids.shape[1] - 1)
    seq = copy_batch(64, g).cuda()
    ids = seq[:, :SPAN + CUE]
    outs = {f: model.generate(ids, max_new_tokens=SPAN - CUE, eos_token_id=[], fp8_weights=f)[:, SPAN + CUE:] for f in (False, True)}
    ppl = {f: math.exp(v / n_tok) for f, v in nll.items()}
    print(json.dumps({"part": "quality", "model": "60m", "train_steps": steps, "ppl_bf16": round(ppl[False], 4),
                      "ppl_fp8": round(ppl[True], 4), "ppl_ratio": round(ppl[True] / ppl[False], 5),
                      "greedy_agreement": round(float((outs[True] == outs[False]).float().mean()), 4),
                      "copy_accuracy_bf16": round(float((outs[False] == seq[:, SPAN + CUE:]).float().mean()), 4),
                      "copy_accuracy_fp8": round(float((outs[True] == seq[:, SPAN + CUE:]).float().mean()), 4)}), flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="kernels,decode,quality")
    ap.add_argument("--models", default="150m,1b")
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--prompts", default="128,1024")
    ap.add_argument("--new-tokens", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--train-steps", type=int, default=1500)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "fp8_weights_bench needs a GPU"
    print(json.dumps(card()), flush=True)
    models = a.models.split(",")
    parts = a.parts.split(",")
    if "kernels" in parts:
        kernels(models, [1, 8, 64])
    if "decode" in parts:
        decode(models, [int(x) for x in a.batches.split(",")], [int(x) for x in a.prompts.split(",")], a.new_tokens, a.reps)
    if "quality" in parts:
        quality(a.train_steps)


if __name__ == "__main__":
    main()
