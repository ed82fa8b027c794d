"""FP8 KV cache on the H100: ``generate(fp8_kv_cache=True)`` against the bf16 cache.

    python profiles/fp8_kv_bench.py                           # every part, one JSON line per measurement
    python profiles/fp8_kv_bench.py --parts attention --models 150m

Parts:

1. ``decode``: 150m and 1b presets (random weights), B in {1, 8, 64}, prompts of 128, 1024 and 1792 random tokens, 256
   new tokens, greedy, no EOS.  Decode ms/token = (time of a 256-token call - time of a 1-token call) / 255, so prefill
   is left out.  bf16 and FP8 caches run on two model objects with the same weights (each keeps its own caches and decode
   graph), each warmed up first, then alternated call by call, --reps times; the minimum is reported, with the cache
   size of each computed from the shapes.
2. ``combined``: the same measurement at B 64 and B 8, prompt 1024, for bf16, the FP8 cache, and the FP8 cache together
   with ``fp8_weights=True``.
3. ``attention``: one layer's decode attention (split-KV kernel + combine) at every decode configuration, on a cache
   filled to the prompt length: CUDA events around one CUDA graph of 200 back-to-back launches, and the K/V bytes read
   computed from the shapes (bf16: 2 * 128 bytes per head-position; FP8: 2 * (64 + 4)).
4. ``quality``: a 60m preset trained here on sequences that repeat a random span (``lookup_bench.py``'s copy task;
   random weights say nothing about quality): greedy agreement between the two caches and copy accuracy of each.
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
from opendiloco_b200.ops import fp8w as FW  # noqa: E402

HBM = 3.35e12


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def cache_gb(cfg, B: int, Smax: int, fp8: bool) -> float:
    per = cfg.head_dim + 4 if fp8 else 2 * cfg.head_dim              # bytes per (layer, K|V, row, kv head, position)
    return cfg.num_hidden_layers * 2 * B * cfg.num_key_value_heads * Smax * per / 1e9


def ms_per_token(calls: dict, new: int, reps: int) -> dict:
    best = {(m, n): math.inf for m in calls for n in (1, new)}
    for m in calls:                                    # warm-up: caches and decode graphs of this shape
        calls[m](new)
        calls[m](1)
    for _ in range(reps):
        for n in (new, 1):
            for m in calls:
                best[m, n] = min(best[m, n], timed_call(lambda: calls[m](n)))
    return {m: (best[m, new] - best[m, 1]) / (new - 1) * 1e3 for m in calls}


def _pair(name: str):
    bf = LlamaForCausalLM(LlamaConfig.from_pretrained(name), device="cuda", precision="bf16-mixed", seed=0).eval()
    f8 = LlamaForCausalLM(LlamaConfig.from_pretrained(name), device="cuda", precision="bf16-mixed", seed=0).eval()
    return bf, f8


def decode(models: list[str], batches: list[int], prompts: list[int], new: int, reps: int) -> None:
    for name in models:
        bf, f8 = _pair(name)
        cfg = bf.config
        for B in batches:
            for P in prompts:
                ids = torch.randint(3, cfg.vocab_size, (B, P), generator=torch.Generator().manual_seed(B + P)).cuda()
                calls = {"bf16": lambda n: bf.generate(ids, max_new_tokens=n, eos_token_id=[]),
                         "fp8_kv": lambda n: f8.generate(ids, max_new_tokens=n, eos_token_id=[], fp8_kv_cache=True)}
                ms = ms_per_token(calls, new, reps)
                agree = float((calls["bf16"](new)[:, P:] == calls["fp8_kv"](new)[:, P:]).float().mean())
                Smax = _round_up(P + new, 128)
                print(json.dumps({"part": "decode", "model": name, "B": B, "prompt": P, "new_tokens": new,
                                  "bf16_ms_per_token": round(ms["bf16"], 4), "fp8_kv_ms_per_token": round(ms["fp8_kv"], 4),
                                  "speedup": round(ms["bf16"] / ms["fp8_kv"], 3),
                                  "bf16_cache_GB": round(cache_gb(cfg, B, Smax, False), 4),
                                  "fp8_kv_cache_GB": round(cache_gb(cfg, B, Smax, True), 4),
                                  "greedy_tokens_equal_bf16": round(agree, 4), "reps": reps}), flush=True)
        del bf, f8
        torch.cuda.empty_cache()


def combined(models: list[str], batches: list[int], P: int, new: int, reps: int) -> None:
    for name in models:
        bf, f8 = _pair(name)
        for B in batches:
            ids = torch.randint(3, bf.config.vocab_size, (B, P), generator=torch.Generator().manual_seed(B + P)).cuda()
            calls = {"bf16": lambda n: bf.generate(ids, max_new_tokens=n, eos_token_id=[]),
                     "fp8_kv": lambda n: f8.generate(ids, max_new_tokens=n, eos_token_id=[], fp8_kv_cache=True),
                     "fp8_kv_fp8_weights": lambda n: f8.generate(ids, max_new_tokens=n, eos_token_id=[], fp8_kv_cache=True,
                                                                 fp8_weights=True)}
            ms = ms_per_token(calls, new, reps)
            print(json.dumps({"part": "combined", "model": name, "B": B, "prompt": P, "new_tokens": new,
                              **{f"{m}_ms_per_token": round(v, 4) for m, v in ms.items()},
                              "speedup_fp8_kv": round(ms["bf16"] / ms["fp8_kv"], 3),
                              "speedup_fp8_kv_fp8_weights": round(ms["bf16"] / ms["fp8_kv_fp8_weights"], 3), "reps": reps}),
                  flush=True)
        del bf, f8
        torch.cuda.empty_cache()


def attention(models: list[str], batches: list[int], prompts: list[int], new: int) -> None:
    for name in models:
        cfg = LlamaConfig.from_pretrained(name)
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        for B in batches:
            for P in prompts:
                Smax = _round_up(P + new, 128)
                g = torch.Generator(device="cuda").manual_seed(B + P)
                kb = torch.randn(B, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
                vb = torch.randn(B, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
                (kq, ki), (vq, vi) = FW.quantize_rows_ref(kb.view(-1, D)), FW.quantize_rows_ref(vb.view(-1, D))
                kq, vq, ki, vi = kq.view(kb.shape), vq.view(vb.shape), ki.view(kb.shape[:-1]), vi.view(vb.shape[:-1])
                q = torch.randn(B, (Hq + 2 * Hkv) * D, device="cuda").bfloat16()
                pos = torch.full((B,), P, dtype=torch.int32, device="cuda")          # the first decode step: P + 1 keys
                nch = DK.attn_chunks(Smax)
                po, pm = torch.empty(B, Hq, nch, D, device="cuda"), torch.empty(B, Hq, nch, 2, device="cuda")
                out = torch.empty(B, Hq * D, dtype=torch.bfloat16, device="cuda")
                t16 = event_time(lambda: DK.attention(q, kb, vb, pos, out, Hq, Hkv, D, po, pm), 200)
                t8 = event_time(lambda: DK.attention(q, kq, vq, pos, out, Hq, Hkv, D, po, pm, kinv=ki, vinv=vi), 200)
                keys = B * Hkv * (P + 1)
                b16, b8 = keys * 2 * D * 2, keys * 2 * (D + 4)
                print(json.dumps({"part": "attention", "model": name, "B": B, "prompt": P, "keys": P + 1,
                                  "bf16_us": round(t16 * 1e6, 2), "fp8_kv_us": round(t8 * 1e6, 2), "speedup": round(t16 / t8, 3),
                                  "bf16_GB_per_s": round(b16 / t16 / 1e9, 1), "fp8_kv_GB_per_s": round(b8 / t8 / 1e9, 1),
                                  "bf16_share_of_hbm": round(b16 / t16 / HBM, 3), "fp8_kv_share_of_hbm": round(b8 / t8 / HBM, 3),
                                  "layers": cfg.num_hidden_layers}), flush=True)
                del kb, vb, kq, vq, ki, vi
        torch.cuda.empty_cache()


def quality(steps: int) -> None:
    from lookup_bench import CUE, SPAN, copy_batch, train_copy_model

    model = train_copy_model(steps, 32, seed=0)
    g = torch.Generator().manual_seed(777)
    seq = copy_batch(64, g).cuda()
    ids = seq[:, :SPAN + CUE]
    outs = {f: model.generate(ids, max_new_tokens=SPAN - CUE, eos_token_id=[], fp8_kv_cache=f)[:, SPAN + CUE:] for f in (False, True)}
    print(json.dumps({"part": "quality", "model": "60m", "train_steps": steps,
                      "greedy_agreement": round(float((outs[True] == outs[False]).float().mean()), 4),
                      "copy_accuracy_bf16": round(float((outs[False] == seq[:, SPAN + CUE:]).float().mean()), 4),
                      "copy_accuracy_fp8_kv": round(float((outs[True] == seq[:, SPAN + CUE:]).float().mean()), 4)}), flush=True)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--parts", default="attention,decode,combined,quality")
    ap.add_argument("--models", default="150m,1b")
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--prompts", default="128,1024,1792")
    ap.add_argument("--new-tokens", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--train-steps", type=int, default=1500)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "fp8_kv_bench needs a GPU"
    print(json.dumps(card()), flush=True)
    models = a.models.split(",")
    parts = a.parts.split(",")
    batches, prompts = [int(x) for x in a.batches.split(",")], [int(x) for x in a.prompts.split(",")]
    if "attention" in parts:
        attention(models, batches, prompts, a.new_tokens)
    if "decode" in parts:
        decode(models, batches, prompts, a.new_tokens, a.reps)
    if "combined" in parts:
        combined(models, [64, 8], 1024, a.new_tokens, a.reps)
    if "quality" in parts:
        quality(a.train_steps)


if __name__ == "__main__":
    main()
