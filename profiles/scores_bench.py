"""Score outputs on the H100: decode ms/token of ``generate`` with ``return_dict_in_generate=True, output_scores=True,
output_logits=True`` against the same calls with the flags off, for greedy decoding, sampling (top_k 50, temperature 0.8)
and beam search (num_beams 4).  Presets with random weights, B in {1, 8}, prompts of 128 tokens, V = 32000, EOS disabled.

    python profiles/scores_bench.py                              # the sweep, one JSON line per configuration
    python profiles/scores_bench.py --models 150m --batches 8

ms/token is the time of one whole ``generate`` call (prefill included; minimum over --reps calls, host clock around a
device synchronise) over its new tokens.  Off and on alternate; the decode state holds one step graph, so each timed
call follows an untimed call of the same flags that allocates the buffers and captures the graph, and the timed call
replays it.  The extra traffic per step is one fp32 and one bf16 row per
live row (beam search: per running beam), 6 * V bytes = 192 KB at V = 32000, written by the sampler (greedy, sampling)
or ``beam_scores_kernel`` (beam search); the returned tuples are copied out of the resident buffers once per call, and
that copy is part of the "on" time.
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

FLAGS = dict(return_dict_in_generate=True, output_scores=True, output_logits=True)
MODES = (("greedy", {}), ("sample", dict(do_sample=True, top_k=50, temperature=0.8)), ("beam", dict(num_beams=4)))


def timed_call(fn) -> float:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="150m,1b")
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--prompt", type=int, default=128)
    ap.add_argument("--new-tokens", type=int, default=128)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "scores_bench needs a GPU"
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
        for B in (int(x) for x in a.batches.split(",")):
            ids = torch.randint(3, V, (B, a.prompt), generator=torch.Generator().manual_seed(B)).cuda()
            row = {"model": name, "B": B, "prompt": a.prompt, "new_tokens": a.new_tokens, "V": V, "reps": a.reps}
            for mode, extra in MODES:
                kw = dict(max_new_tokens=a.new_tokens, eos_token_id=[], seed=1, **extra)
                calls = {"off": lambda: model.generate(ids, **kw), "on": lambda: model.generate(ids, **kw, **FLAGS)}
                t = {"off": [], "on": []}
                for _ in range(a.reps):                  # alternating rounds; the state keeps one step graph, so each
                    for s in ("off", "on"):              # timed call follows an untimed one that captures it
                        calls[s]()
                        t[s].append(timed_call(calls[s]))
                for s in ("off", "on"):
                    row[f"{mode}_ms_per_token_{s}"] = round(1e3 * min(t[s]) / a.new_tokens, 4)
                row[f"{mode}_overhead_pct"] = round(100 * (min(t["on"]) / min(t["off"]) - 1), 2)
                model.engine.beam_state = None
                model.engine.decode_state = None
                torch.cuda.empty_cache()
            emit(row)
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
