"""Logits processors on the H100: decode ms/token and beam-step time of ``generate`` with ``no_repeat_ngram_size=3`` and
``repetition_penalty=1.2`` against the same calls with the processors off, and the sampler / beam_topk kernels' own time.
Presets with random weights, B in {1, 8, 64}, prompts of 128 and 1024 tokens, EOS disabled.

    python profiles/processors_bench.py                          # the sweep, one JSON line per configuration
    python profiles/processors_bench.py --models 150m --batches 8 --prompts 128
    python profiles/processors_bench.py --processors sequence   # sequence_bias, bad_words_ids and min_length instead

``--processors sequence`` times 200 ``bad_words_ids`` of 1-4 random ids, 50 ``sequence_bias`` entries of 1-3 ids and
``min_length=64`` (a sequence table of 250 entries, matched against every row's history each step) instead of the
repetition controls; the rows and their columns are the same.

ms/token is the time of one whole ``generate`` call (prefill included; minimum over --reps calls, host clock around a
device synchronise) over its new tokens; each mode is timed after a warm-up call of the same mode and shape, and off
and on alternate.  Beam search runs num_beams = 4 on the same prompts.  The kernel times come from ``torch.profiler``
over --profile-steps eager steps in a separate pass: ``sample_kernel`` for greedy decode, ``beam_topk_kernel`` +
``beam_step_kernel`` for beam search.  The history the processors read is B * (P + generated) int32 per step.
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
from opendiloco_b200.models.generation import beam_step, step  # noqa: E402
from opendiloco_b200.models.llama import LlamaForCausalLM  # noqa: E402

PROC = dict(no_repeat_ngram_size=3, repetition_penalty=1.2)
OFF = dict(no_repeat_ngram_size=0, repetition_penalty=1.0)


def sequence_processors(V: int, seed: int = 0) -> dict:
    """200 bad words of 1-4 ids, 50 sequence biases of 1-3 ids and min_length 64, drawn from a fixed seed."""
    g = torch.Generator().manual_seed(seed)
    ids = lambda n: torch.randint(3, V, (n,), generator=g).tolist()   # noqa: E731
    bad = [ids(1 + i % 4) for i in range(200)]
    bias = {tuple(ids(1 + i % 3)): float(torch.randn((), generator=g) * 2) for i in range(50)}
    return dict(bad_words_ids=bad, sequence_bias=bias, min_length=64)


def timed_call(fn) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def kernel_us(fn, names: tuple, steps: int) -> float:
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    us = sum(e.device_time for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and any(k in e.name for k in names))
    return us / steps


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="150m,1b")
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--prompts", default="128,1024")
    ap.add_argument("--new-tokens", type=int, default=128)
    ap.add_argument("--num-beams", type=int, default=4)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--profile-steps", type=int, default=20)
    ap.add_argument("--processors", choices=["repetition", "sequence"], default="repetition",
                    help="repetition: no_repeat_ngram_size=3, repetition_penalty=1.2; sequence: see the module docstring")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "processors_bench needs a GPU"
    sink = open(a.out, "a") if a.out else None

    def emit(row):
        print(json.dumps(row), flush=True)
        if sink:
            sink.write(json.dumps(row) + "\n")
            sink.flush()

    emit(card())
    for name in a.models.split(","):
        model = LlamaForCausalLM(LlamaConfig.from_pretrained(name), device="cuda", precision="bf16-mixed", seed=0).eval()
        V = model.config.vocab_size
        on = PROC if a.processors == "repetition" else sequence_processors(V)
        off = OFF if a.processors == "repetition" else {}
        for P in (int(x) for x in a.prompts.split(",")):
            for B in (int(x) for x in a.batches.split(",")):
                ids = torch.randint(3, V, (B, P), generator=torch.Generator().manual_seed(B + P)).cuda()
                row = {"model": name, "B": B, "prompt": P, "new_tokens": a.new_tokens, "num_beams": a.num_beams, "reps": a.reps}
                if a.processors != "repetition":
                    row["processors"] = a.processors
                for mode, extra in (("greedy", {}), ("beam", dict(num_beams=a.num_beams))):
                    kw = dict(max_new_tokens=a.new_tokens, eos_token_id=[], **extra)
                    t = {"off": [], "on": []}
                    for s, p in (("off", off), ("on", on)):
                        model.generate(ids, **kw, **p)                         # warm-up: caches and step graph of this shape
                    for _ in range(a.reps):
                        for s, p in (("off", off), ("on", on)):
                            t[s].append(timed_call(lambda: model.generate(ids, **kw, **p)))
                    for s in ("off", "on"):
                        row[f"{mode}_ms_per_token_{s}"] = round(1e3 * min(t[s]) / a.new_tokens, 3)
                    for s, p in (("off", off), ("on", on)):
                        model.generate(ids, **dict(kw, max_new_tokens=a.new_tokens // 2), **p)   # leaves the state mid-run
                        if mode == "greedy":
                            st = model.engine.decode_state
                            us = kernel_us(lambda: step(model, st, graph=False), ("sample_kernel",), a.profile_steps)
                            row[f"sampler_us_{s}"] = round(us, 2)
                        else:
                            bs = model.engine.beam_state
                            us = kernel_us(lambda: beam_step(model, bs, 1.0, 0, graph=False), ("beam_topk_kernel", "beam_step_kernel"),
                                           a.profile_steps)
                            row[f"beam_select_us_{s}"] = round(us, 2)
                row["history_MB_per_step_at_end"] = round(B * (P + a.new_tokens) * 4 / 1e6, 3)
                emit(row)
                model.engine.beam_state = None
                model.engine.decode_state = None
                torch.cuda.empty_cache()
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
