"""Beam search on the H100: new tokens/s of ``generate(num_beams=...)`` against greedy ``generate`` on the same number of
rows, the per-step time of the selection and reorder kernels, and the K/V bytes the chunk table saves.  Llama-1B preset
with random weights, B in {1, 8}, num_beams in {4, 8}, a 128-token prompt, 256 new tokens, EOS disabled.

    python profiles/beam_bench.py                       # the sweep, one JSON line per configuration
    python profiles/beam_bench.py --batches 1 --beams 4

Rates count decoded rows: B * num_beams * new_tokens over the time of one whole ``generate`` call (prefill included;
minimum over --reps calls, host clock around a device synchronise), greedy on B * num_beams prompts for comparison.
Each mode is timed after a warm-up call of the same mode and shape.  The kernel times come from ``torch.profiler`` over
--profile-steps eager beam steps in a separate pass.  The byte counts come from a third pass that reads the parents and
positions after every step: ``beam_reorder`` copies the partial 128-position chunk of every beam whose parent is another
row, while a full reorder (as transformers does) copies every beam's whole cache.  EOS is disabled, so every call runs
all steps.
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
from opendiloco_b200.models.generation import beam_prefill, beam_select, beam_state, beam_step  # noqa: E402
from opendiloco_b200.models.llama import LlamaForCausalLM  # noqa: E402
from opendiloco_b200.ops import decode as DK  # noqa: E402

SELECT_KERNELS = ("beam_topk_kernel", "beam_step_kernel", "beam_reorder_kernel")


def timed_call(fn) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def _fresh_state(model, ids, nb: int, n_new: int):
    B, P = ids.shape
    bs = beam_state(model, B, nb, DK.beams_to_keep(nb, 0), n_new, (P + n_new + 127) // 128 * 128)
    bs.dec.set_controls(False, 1.0, 0, 1.0, 0, 0, [])
    bs.reset(0)
    beam_prefill(model, bs, ids, torch.full((B,), P, dtype=torch.int32, device="cuda"))
    beam_select(bs, 1.0, 0)
    return bs


def kernel_us_per_step(model, ids, nb: int, n_new: int, steps: int) -> float:
    from torch.profiler import ProfilerActivity, profile

    bs = _fresh_state(model, ids, nb, n_new)
    beam_step(model, bs, 1.0, 0, graph=False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            beam_step(model, bs, 1.0, 0, graph=False)
        torch.cuda.synchronize()
    us = sum(e.device_time for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
             and any(k in e.name for k in SELECT_KERNELS))
    return us / steps


def reorder_bytes(model, ids, nb: int, n_new: int) -> tuple[int, int]:
    """(bytes beam_reorder copied, bytes a whole-cache reorder would copy) over one generate's steps."""
    cfg = model.config
    per_pos = cfg.num_hidden_layers * 2 * cfg.num_key_value_heads * cfg.head_dim * 2      # K and V of one position, bf16
    bs = _fresh_state(model, ids, nb, n_new)
    ours = full = 0
    for t in range(n_new):
        if t:
            beam_step(model, bs, 1.0, 0)
        rows = torch.arange(bs.parent.numel(), device="cuda")
        moved = bs.parent.long() != rows
        pos = bs.dec.pos.long()
        ours += int(((pos % 128) * moved).sum()) * per_pos
        full += int(pos.sum()) * per_pos
    return ours, full


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="1b")
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--beams", default="4,8")
    ap.add_argument("--prompt", type=int, default=128)
    ap.add_argument("--new-tokens", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=20)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "beam_bench needs a GPU"
    print(json.dumps(card()), flush=True)
    model = LlamaForCausalLM(LlamaConfig.from_pretrained(a.model), device="cuda", precision="bf16-mixed", seed=0).eval()
    V = model.config.vocab_size
    for B in (int(x) for x in a.batches.split(",")):
        ids = torch.randint(3, V, (B, a.prompt), generator=torch.Generator().manual_seed(B)).cuda()
        for nb in (int(x) for x in a.beams.split(",")):
            rows = B * nb
            kw = dict(max_new_tokens=a.new_tokens, eos_token_id=[])
            many = ids.repeat_interleave(nb, dim=0)
            model.generate(many, **kw)                      # warm-up: caches and decode graph of this shape
            tg = min(timed_call(lambda: model.generate(many, **kw)) for _ in range(a.reps))
            bkw = dict(kw, num_beams=nb, num_return_sequences=nb)
            model.generate(ids, **bkw)                      # warm-up: beam caches and step graph of this shape
            tb = min(timed_call(lambda: model.generate(ids, **bkw)) for _ in range(a.reps))
            us = kernel_us_per_step(model, ids, nb, a.new_tokens, a.profile_steps)
            ours, full = reorder_bytes(model, ids, nb, a.new_tokens)
            row = {"model": a.model, "B": B, "num_beams": nb, "rows": rows, "prompt": a.prompt, "new_tokens": a.new_tokens,
                   "greedy_tokens_per_s": round(rows * a.new_tokens / tg, 1), "beam_tokens_per_s": round(rows * a.new_tokens / tb, 1),
                   "beam_over_greedy": round(tg / tb, 3), "select_reorder_us_per_step": round(us, 1),
                   "reorder_kv_MB": round(ours / 1e6, 1), "full_reorder_kv_MB": round(full / 1e6, 1), "reps": a.reps}
            print(json.dumps(row), flush=True)
            model.engine.beam_state = None
            model.engine.decode_state = None
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
