"""Assisted (speculative) generation on the H100: tokens/s of ``generate(assistant_model=...)`` against plain ``generate``
for a Llama-1B target, with the 150M preset or the target itself as the draft, B in {1, 8}, K in {2, 4, 6}.

    python profiles/assisted_bench.py                       # the sweep, one JSON line per configuration
    python profiles/assisted_bench.py --drafts self --batches 1 --ks 4

Weights are random from a seed, so a distinct draft agrees with the target on almost nothing: its acceptance is near
zero and its rows measure the cost of a round that emits one token.  The self-draft rows (acceptance ~1 up to bf16
near-ties) bound the verify path's overhead from the other side.  The speedup on a trained checkpoint pair depends on
its acceptance rate and is not measured here.

Greedy decoding, no EOS.  A timing is the minimum over --reps whole ``generate`` calls (prefill included; host clock
around a device synchronise).  Each mode is timed after a warm-up call of the same mode and configuration, with no other
call in between: plain and assisted ``generate`` size their caches differently (assisted adds K positions), so
alternating them would reallocate the caches and recapture the CUDA graphs inside every timed call.
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


def timed_call(fn) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--target", default="1b")
    ap.add_argument("--drafts", default="150m,self")
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--ks", default="2,4,6")
    ap.add_argument("--prompt", type=int, default=128)
    ap.add_argument("--new-tokens", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "assisted_bench needs a GPU"
    print(json.dumps(card()), flush=True)
    target = LlamaForCausalLM(LlamaConfig.from_pretrained(a.target), device="cuda", precision="bf16-mixed", seed=0).eval()
    V = target.config.vocab_size
    for dname in a.drafts.split(","):
        draft = target if dname == "self" else \
            LlamaForCausalLM(LlamaConfig.from_pretrained(dname), device="cuda", precision="bf16-mixed", seed=1).eval()
        for B in (int(x) for x in a.batches.split(",")):
            ids = torch.randint(3, V, (B, a.prompt), generator=torch.Generator().manual_seed(B)).cuda()
            kw = dict(max_new_tokens=a.new_tokens, eos_token_id=[])
            plain_out = target.generate(ids, **kw)           # warm-up: caches and decode graph of this shape
            tp = min(timed_call(lambda: target.generate(ids, **kw)) for _ in range(a.reps))
            for Kp in (int(x) for x in a.ks.split(",")):
                akw = dict(kw, assistant_model=draft, num_assistant_tokens=Kp)
                out = target.generate(ids, **akw)            # warm-up: caches and round graph of this shape
                st = target.engine.assisted_state
                acc, passes = st.acceptance_rate(), st.verify_passes()
                same = float((out[:, a.prompt:] == plain_out[:, a.prompt:]).float().mean())
                ta = min(timed_call(lambda: target.generate(ids, **akw)) for _ in range(a.reps))
                row = {"target": a.target, "draft": dname, "B": B, "K": Kp, "prompt": a.prompt, "new_tokens": a.new_tokens,
                       "plain_tokens_per_s": round(B * a.new_tokens / tp, 1), "assisted_tokens_per_s": round(B * a.new_tokens / ta, 1),
                       "speedup": round(tp / ta, 3), "acceptance": round(acc, 4), "verify_passes": passes,
                       "tokens_equal_plain": round(same, 4), "reps": a.reps}
                print(json.dumps(row), flush=True)
        del draft
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
