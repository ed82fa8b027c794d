"""Multi-sample generation on the H100: ``generate(do_sample=True, num_return_sequences=n)`` against the repeated-prompt
call ``generate(ids.repeat_interleave(n, 0), ...)``.

    python profiles/multi_sample_bench.py                     # both parts, one JSON line per measurement
    python profiles/multi_sample_bench.py --parts kernel --models 150m

Parts:

1. ``e2e``: 150m and 1b presets (random weights), B in {1, 8} prompts of 512 and 1024 random tokens, n in {8, 16}
   samples each, 256 new tokens, ``do_sample=True``, no EOS.  The two programs run on two model objects with the same
   weights (each keeps its own caches and decode graph); every shape is warmed up, then the calls alternate, --reps
   rounds, and the minimum is reported.  Prefill ms = the time of a 1-token call; decode ms/token = (time of the 256-token
   call - time of the 1-token call) / 255; tokens/s = B * n * 256 / time of the 256-token call.  Peak memory: the peak
   allocated bytes of one call above what was allocated before it, starting with no decode state (so the caches, the
   prefill buffers and the transient activations all count).
2. ``kernel``: B in {1, 8, 32}, prompts of 512, 1024 and 1792: one layer's decode attention on the cache of the first
   decode step after a fork (rows = B * n, every sibling at position P, the prompt's complete chunks shared through the
   chunk table): ``attention`` through the table (one CTA per row and chunk) against ``attention_grouped`` (one load per
   shared chunk and CTA, at the launcher's sibling split, and at forced splits).  CUDA events around one CUDA graph of
   200 launches each.  Unique bytes are the K/V bytes the table names, computed from the shapes: the shared chunks once
   per prompt, each row's own keys once per row.
"""
from __future__ import annotations

import argparse
import json
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from fp8_weights_bench import event_time, timed_call  # noqa: E402
from generate_bench import card  # noqa: E402
from opendiloco_b200.models.config import LlamaConfig  # noqa: E402
from opendiloco_b200.models.llama import LlamaForCausalLM  # noqa: E402
from opendiloco_b200.ops import decode as DK  # noqa: E402

HBM = 3.35e12


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def peak_bytes(model, fn) -> int:
    model.engine.decode_state = None
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def e2e(models: list[str], batches: list[int], prompts: list[int], ns: list[int], new: int, reps: int) -> None:
    for name in models:
        cfg = LlamaConfig.from_pretrained(name)
        pair = {k: LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=0).eval() for k in ("multi", "repeated")}
        for B in batches:
            for P in prompts:
                ids = torch.randint(3, cfg.vocab_size, (B, P), generator=torch.Generator().manual_seed(B + P)).cuda()
                for n in ns:
                    kw = dict(do_sample=True, eos_token_id=[], seed=1)
                    rep = ids.repeat_interleave(n, 0)
                    calls = {"multi": lambda t: pair["multi"].generate(ids, max_new_tokens=t, num_return_sequences=n, **kw),
                             "repeated": lambda t: pair["repeated"].generate(rep, max_new_tokens=t, **kw)}
                    peak = {k: peak_bytes(pair[k], lambda: calls[k](new)) for k in calls}
                    same = torch.equal(calls["multi"](new), calls["repeated"](new))
                    best = {(k, t): math.inf for k in calls for t in (1, new)}
                    for k in calls:                                # warm-up of both lengths (graphs captured above)
                        calls[k](1)
                    for _ in range(reps):
                        for t in (new, 1):
                            for k in calls:
                                best[k, t] = min(best[k, t], timed_call(lambda: calls[k](t)))
                    res = {}
                    for k in calls:
                        res[f"{k}_prefill_ms"] = round(best[k, 1] * 1e3, 3)
                        res[f"{k}_decode_ms_per_token"] = round((best[k, new] - best[k, 1]) / (new - 1) * 1e3, 4)
                        res[f"{k}_tokens_per_s"] = round(B * n * new / best[k, new], 1)
                        res[f"{k}_peak_GB"] = round(peak[k] / 1e9, 3)
                    print(json.dumps({"part": "e2e", "model": name, "B": B, "prompt": P, "n": n, "new_tokens": new, **res,
                                      "prefill_speedup": round(best["repeated", 1] / best["multi", 1], 3),
                                      "decode_speedup": round(res["repeated_decode_ms_per_token"] / res["multi_decode_ms_per_token"], 3),
                                      "tokens_equal": same, "reps": reps}), flush=True)
        del pair
        torch.cuda.empty_cache()


def kernel(models: list[str], batches: list[int], prompts: list[int], ns: list[int], new: int, fp8: bool) -> None:
    for name in models:
        cfg = LlamaConfig.from_pretrained(name)
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        for B in batches:
            for P in prompts:
                for n in ns:
                    rows, Smax = B * n, _round_up(P + new, 128)
                    g = torch.Generator(device="cuda").manual_seed(B + P + n)
                    if fp8:
                        kc = torch.randint(0, 120, (rows, Hkv, Smax, D), device="cuda", dtype=torch.uint8, generator=g)
                        vc = torch.randint(0, 120, (rows, Hkv, Smax, D), device="cuda", dtype=torch.uint8, generator=g)
                        kc, vc = kc.view(torch.float8_e4m3fn), vc.view(torch.float8_e4m3fn)
                        ki = torch.full((rows, Hkv, Smax), 2.0 ** -4, device="cuda")
                        vi = ki.clone()
                    else:
                        kc = torch.randn(rows, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
                        vc = torch.randn(rows, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
                        ki = vi = None
                    c = P // 128                                  # the fork at P: chunks < c shared, the rest each row's own
                    r = torch.arange(rows, dtype=torch.int32, device="cuda")
                    table = torch.where(torch.arange(Smax // 128, device="cuda")[None, :] < c, (r // n * n)[:, None], r[:, None])
                    table = table.to(torch.int32).contiguous()
                    q = torch.randn(rows, (Hq + 2 * Hkv) * D, device="cuda").bfloat16()
                    pos = torch.full((rows,), P, dtype=torch.int32, device="cuda")
                    nch = DK.attn_chunks(Smax)
                    po, pm = torch.empty(rows, Hq, nch, D, device="cuda"), torch.empty(rows, Hq, nch, 2, device="cuda")
                    a, b = (torch.empty(rows, Hq * D, dtype=torch.bfloat16, device="cuda") for _ in range(2))
                    t_tab = event_time(lambda: DK.attention(q, kc, vc, pos, a, Hq, Hkv, D, po, pm, table=table, kinv=ki, vinv=vi), 200)
                    t_grp = event_time(lambda: DK.attention_grouped(q, kc, vc, pos, b, Hq, Hkv, D, n, po, pm, table=table, kinv=ki,
                                                                    vinv=vi), 200)
                    assert torch.equal(a, b)
                    grouped = lambda s: DK.attention_grouped(q, kc, vc, pos, b, Hq, Hkv, D, n, po, pm, table=table,  # noqa: E731
                                                             kinv=ki, vinv=vi, splits=s)
                    sweep = {s: round(event_time(lambda: grouped(s), 200) * 1e6, 2) for s in sorted({1, 2, 4, 8, n}) if s <= n}
                    per_key = Hkv * 2 * (D + 4 if fp8 else 2 * D)
                    unique = per_key * (B * 128 * c + rows * (P + 1 - 128 * c))
                    print(json.dumps({"part": "kernel", "model": name, "cache": "fp8" if fp8 else "bf16", "B": B, "prompt": P, "n": n,
                                      "keys": P + 1, "splits": DK.attn_group_splits(rows, n, Hq, Hkv, Smax, fp8),
                                      "table_us": round(t_tab * 1e6, 2), "grouped_us": round(t_grp * 1e6, 2),
                                      "speedup": round(t_tab / t_grp, 3), "grouped_us_by_splits": sweep,
                                      "unique_MB": round(unique / 1e6, 2),
                                      "table_unique_GB_per_s": round(unique / t_tab / 1e9, 1),
                                      "grouped_unique_GB_per_s": round(unique / t_grp / 1e9, 1),
                                      "repeated_MB": round(per_key * rows * (P + 1) / 1e6, 2), "layers": cfg.num_hidden_layers}),
                          flush=True)
                    del kc, vc, ki, vi
        torch.cuda.empty_cache()


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="kernel,e2e")
    ap.add_argument("--models", default="150m,1b")
    ap.add_argument("--batches", default="1,8")
    ap.add_argument("--kernel-batches", default="1,8,32", help="kernel part: prompts per call")
    ap.add_argument("--kernel-prompts", default="512,1024,1792", help="kernel part: prompt lengths")
    ap.add_argument("--prompts", default="512,1024")
    ap.add_argument("--ns", default="8,16")
    ap.add_argument("--new-tokens", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--fp8-kv", action="store_true", help="kernel part: the FP8 cache")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "multi_sample_bench needs a GPU"
    print(json.dumps(card()), flush=True)
    models, parts = a.models.split(","), a.parts.split(",")
    batches, prompts, ns = ([int(x) for x in s.split(",")] for s in (a.batches, a.prompts, a.ns))
    if "kernel" in parts:
        kernel(models, [int(x) for x in a.kernel_batches.split(",")], [int(x) for x in a.kernel_prompts.split(",")], ns, a.new_tokens,
               a.fp8_kv)
    if "e2e" in parts:
        e2e(models, batches, prompts, ns, a.new_tokens, a.reps)


if __name__ == "__main__":
    main()
