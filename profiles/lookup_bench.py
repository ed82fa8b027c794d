"""Prompt lookup decoding on the H100: tokens/s of ``generate(prompt_lookup_num_tokens=K)`` against plain ``generate``.

    python profiles/lookup_bench.py                         # both parts, one JSON line per configuration
    python profiles/lookup_bench.py --part overhead --models 150m --batches 8 --ks 4

Two parts:

1. ``overhead``: the 150m and 1b presets with random weights and random prompts.  Random prompts hold no useful
   matches, so rounds that find none emit one token each and measure the cost of a lookup round (proposal kernel +
   verify pass over (K+1)*B rows + acceptance) against one decode step.  A random model whose greedy output falls into a
   loop gets matches from the loop; the acceptance column shows how much.
2. ``copy``: a 60m preset trained here, through the project's trainer, on sequences that repeat a random span (x x, x
   128 random tokens from a 1021-token alphabet).  Its prompts are x followed by the first 16 tokens of x again, so the
   continuation is the rest of x: the trained model's greedy copy accuracy is reported, then lookup is timed against
   plain decoding on those prompts.

Greedy decoding, no EOS.  A timing is the minimum over --reps whole ``generate`` calls (prefill included; host clock
around a device synchronise).  Each mode is timed after a warm-up call of the same mode and configuration, with no other
call in between: plain and lookup ``generate`` size their caches differently (lookup adds K positions), so alternating
them would reallocate the caches and recapture the CUDA graphs inside every timed call.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from generate_bench import card  # noqa: E402
from opendiloco_b200.models.config import LlamaConfig  # noqa: E402
from opendiloco_b200.models.llama import LlamaForCausalLM  # noqa: E402

SPAN = 128                     # copy workload: the repeated span
CUE = 16                       # copy workload: tokens of the second copy given in the prompt
ALPHABET = 1024                # copy workload: span tokens are drawn from ids [3, 1024)


def timed_call(fn) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def compare(model, ids, new_tokens: int, ks: list[int], reps: int, label: dict) -> None:
    """One JSON line per K: plain and lookup tokens/s, acceptance, verify passes, agreement with plain greedy."""
    B, P = ids.shape
    kw = dict(max_new_tokens=new_tokens, eos_token_id=[])
    plain_out = model.generate(ids, **kw)                 # warm-up: caches and decode graph of this shape
    tp = min(timed_call(lambda: model.generate(ids, **kw)) for _ in range(reps))
    for K in ks:
        lkw = dict(kw, prompt_lookup_num_tokens=K)
        out = model.generate(ids, **lkw)                  # warm-up: caches and round graph of this shape
        st = model.engine.assisted_state
        acc, passes = st.acceptance_rate(), st.verify_passes()
        proposed = int(st.proposed.sum()) / B
        same = float((out[:, P:] == plain_out[:, P:]).float().mean())
        tl = min(timed_call(lambda: model.generate(ids, **lkw)) for _ in range(reps))
        row = dict(label, B=B, K=K, prompt=P, new_tokens=new_tokens, plain_tokens_per_s=round(B * new_tokens / tp, 1),
                   lookup_tokens_per_s=round(B * new_tokens / tl, 1), speedup=round(tp / tl, 3), acceptance=round(acc, 4),
                   proposed_per_row=round(proposed, 1), verify_passes=passes, tokens_equal_plain=round(same, 4), reps=reps)
        print(json.dumps(row), flush=True)


def copy_batch(B: int, g: torch.Generator) -> torch.Tensor:
    x = torch.randint(3, ALPHABET, (B, SPAN), generator=g)
    return torch.cat([x, x], dim=1)


def train_copy_model(steps: int, batch: int, seed: int) -> LlamaForCausalLM:
    from opendiloco_b200.trainer import DiLoCoTrainer, TrainerConfig

    model = LlamaForCausalLM(LlamaConfig.from_pretrained("60m"), device="cuda", precision="bf16-mixed", seed=seed)
    tr = DiLoCoTrainer(model, TrainerConfig(lr=1e-3, warmup_steps=50, total_steps=steps, local_steps=None, samples_per_step=batch))
    g = torch.Generator().manual_seed(seed)

    def batches():
        while True:
            ids = copy_batch(batch, g)
            yield {"input_ids": ids, "labels": ids}

    it = batches()
    t0 = time.perf_counter()
    for s in range(steps):
        loss = tr.train_step(it)
        if (s + 1) % 500 == 0:
            print(json.dumps({"train_step": s + 1, "loss": round(float(loss), 4),
                              "seconds": round(time.perf_counter() - t0, 1)}), flush=True)
    return model.eval()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--part", choices=["overhead", "copy", "both"], default="both")
    ap.add_argument("--models", default="150m,1b")
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--ks", default="2,4,7")
    ap.add_argument("--prompt", type=int, default=128)
    ap.add_argument("--new-tokens", type=int, default=128)
    ap.add_argument("--train-steps", type=int, default=3000)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "lookup_bench needs a GPU"
    print(json.dumps(card()), flush=True)
    ks = [int(x) for x in a.ks.split(",")]
    batches = [int(x) for x in a.batches.split(",")]
    if a.part in ("overhead", "both"):
        for name in a.models.split(","):
            model = LlamaForCausalLM(LlamaConfig.from_pretrained(name), device="cuda", precision="bf16-mixed", seed=0).eval()
            for B in batches:
                ids = torch.randint(3, model.config.vocab_size, (B, a.prompt), generator=torch.Generator().manual_seed(B)).cuda()
                compare(model, ids, a.new_tokens, ks, a.reps, {"part": "overhead", "model": name})
            del model
            torch.cuda.empty_cache()
    if a.part in ("copy", "both"):
        model = train_copy_model(a.train_steps, 32, seed=0)
        g = torch.Generator().manual_seed(12345)
        new = SPAN - CUE
        for B in batches:
            seq = copy_batch(B, g).cuda()
            ids = seq[:, :SPAN + CUE]
            out = model.generate(ids, max_new_tokens=new, eos_token_id=[])
            accuracy = float((out[:, SPAN + CUE:] == seq[:, SPAN + CUE:]).float().mean())
            compare(model, ids, new, ks, a.reps, {"part": "copy", "model": "60m", "train_steps": a.train_steps,
                                                  "greedy_copy_accuracy": round(accuracy, 4)})


if __name__ == "__main__":
    main()
