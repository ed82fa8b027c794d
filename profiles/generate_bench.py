"""KV-cached generation on the H100: prefill time, decode ms/token and tokens/s, decode-attention KV-read bandwidth, and
end-to-end ``generate`` against transformers ``generate`` (bf16, same weights, same GPU, alternated in one process).

    python profiles/generate_bench.py                       # the sweep: presets 150m, 1b x B {1, 8, 64} x prompt {128, 1024}
    python profiles/generate_bench.py --profile             # per-kernel breakdown of one eager decode step (torch.profiler)

Weights are random from a seed.  Every timing uses CUDA events around work repeated for at least --window seconds after
a warm-up.  The profile run writes its table and trace under profiles_out/.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from opendiloco_b200.models.config import LlamaConfig  # noqa: E402
from opendiloco_b200.models.generation import decode_state, prefill, step  # noqa: E402
from opendiloco_b200.models.llama import LlamaForCausalLM  # noqa: E402
from opendiloco_b200.ops import decode as DK  # noqa: E402

OUT_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "profiles_out")


def card() -> dict:
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["max_sm_clock"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # noqa: BLE001
        info["power_limit"] = f"unknown ({e})"
    return info


def timed(fn, window: float, min_reps: int = 3) -> float:
    """Mean seconds per call of fn over >= window seconds (CUDA events), after one warm-up call."""
    fn()
    torch.cuda.synchronize()
    reps, total = 0, 0.0
    while total < window or reps < min_reps:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        total += a.elapsed_time(b) / 1e3
        reps += 1
    return total / reps


def hf_model(ours: LlamaForCausalLM, device="cuda"):
    """transformers LlamaForCausalLM in bf16 holding our weights (built from our config, state dict copied over)."""
    import transformers as tr

    d = ours.config.to_dict()
    cfg = tr.LlamaConfig(**{k: v for k, v in d.items() if k not in ("architectures", "model_type")})
    m = tr.LlamaForCausalLM(cfg).to(torch.bfloat16)
    m.load_state_dict({n: ours.arena.p(n).detach().cpu() for n, _ in ours.named_parameters()})
    return m.to(device).eval()


def bench_preset(name: str, batches, prompts, new: int, window: float, with_hf: bool) -> list[dict]:
    cfg = LlamaConfig.from_pretrained(name)
    model = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=0)
    hf = hf_model(model) if with_hf else None
    rows = []
    L, Hkv, D = cfg.num_hidden_layers, cfg.num_key_value_heads, cfg.head_dim
    for B in batches:
        for P in prompts:
            g = torch.Generator().manual_seed(B * 10007 + P)
            ids = torch.randint(3, cfg.vocab_size, (B, P), generator=g).cuda()
            Smax = (P + new + 127) // 128 * 128
            st = decode_state(model, B, Smax)
            st.set_controls(False, 1.0, 0, 1.0, 0, 0, [])
            lens = torch.full((B,), P, dtype=torch.int32, device="cuda")
            Sp = (P + 127) // 128 * 128
            comp = torch.zeros(B, Sp, dtype=torch.int64, device="cuda")
            comp[:, :P] = ids
            t_prefill = timed(lambda: prefill(model, st, comp, lens), window)

            def decode_all():
                prefill(model, st, comp, lens)
                for _ in range(new - 1):
                    step(model, st)

            t_all = timed(decode_all, window)
            ms_tok = (t_all - t_prefill) / (new - 1) * 1e3
            # decode attention alone at the mean context of the run, one layer's cache
            ctx = P + new // 2
            prefill(model, st, comp, lens)
            st.pos.fill_(ctx - 1)
            t_att = timed(lambda: [DK.attention(st.qkv, st.kc[0], st.vc[0], st.pos, st.att, cfg.num_attention_heads, Hkv, D,
                                                st.part_o, st.part_ml) for _ in range(100)], window) / 100
            kv_bytes = B * Hkv * ctx * D * 2 * 2                          # K and V, bf16
            row = {"preset": name, "B": B, "prompt": P, "new_tokens": new, "prefill_ms": round(t_prefill * 1e3, 3),
                   "decode_ms_per_token": round(ms_tok, 4), "decode_tokens_per_s": round(B / ms_tok * 1e3, 1),
                   "attn_us_per_layer": round(t_att * 1e6, 2), "attn_ctx": ctx, "attn_kv_read_GBps": round(kv_bytes / t_att / 1e9, 1),
                   "decode_attn_share_est": round(t_att * L / (ms_tok / 1e3), 3)}
            if hf is not None:
                mask = torch.ones_like(ids)
                ours_e2e, hf_e2e = [], []
                gen_kw = dict(max_new_tokens=new, eos_token_id=[])
                model.generate(ids, attention_mask=mask, **gen_kw)
                with torch.no_grad():
                    hf.generate(ids, attention_mask=mask, max_new_tokens=new, min_new_tokens=new, do_sample=False, pad_token_id=0)
                t_end = time.time() + 2 * window
                while time.time() < t_end or len(ours_e2e) < 2:          # alternate the two implementations
                    ours_e2e.append(timed(lambda: model.generate(ids, attention_mask=mask, **gen_kw), 0, 1))
                    with torch.no_grad():
                        hf_e2e.append(timed(lambda: hf.generate(ids, attention_mask=mask, max_new_tokens=new, min_new_tokens=new,
                                                                do_sample=False, pad_token_id=0), 0, 1))
                row.update(ours_generate_s=round(min(ours_e2e), 4), hf_generate_s=round(min(hf_e2e), 4),
                           speedup_vs_hf=round(min(hf_e2e) / min(ours_e2e), 2), reps=len(ours_e2e))
            print(json.dumps(row), flush=True)
            rows.append(row)
            model.engine.decode_state = None
    return rows


def profile_step(name: str, B: int, P: int) -> None:
    from torch.profiler import ProfilerActivity, profile

    cfg = LlamaConfig.from_pretrained(name)
    model = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=0)
    st = decode_state(model, B, (P + 256 + 127) // 128 * 128)
    st.set_controls(False, 1.0, 0, 1.0, 0, 0, [])
    ids = torch.randint(3, cfg.vocab_size, (B, P), device="cuda")
    Sp = (P + 127) // 128 * 128
    comp = torch.zeros(B, Sp, dtype=torch.int64, device="cuda")
    comp[:, :P] = ids
    prefill(model, st, comp, torch.full((B,), P, dtype=torch.int32, device="cuda"))
    for _ in range(3):
        step(model, st, graph=False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step(model, st, graph=False)
        torch.cuda.synchronize()
    os.makedirs(OUT_DIR, exist_ok=True)
    tag = f"decode_step_{name}_B{B}_P{P}"
    table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=30)
    with open(os.path.join(OUT_DIR, tag + ".txt"), "w") as f:
        f.write(json.dumps(card()) + "\n" + table + "\n")
    prof.export_chrome_trace(os.path.join(OUT_DIR, tag + ".pt.trace.json"))
    print(tag)
    print(table)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--presets", default="150m,1b")
    ap.add_argument("--batches", default="1,8,64")
    ap.add_argument("--prompts", default="128,1024")
    ap.add_argument("--new-tokens", type=int, default=256)
    ap.add_argument("--window", type=float, default=1.0, help="seconds of timed work per number")
    ap.add_argument("--no-hf", action="store_true", help="skip the transformers comparison")
    ap.add_argument("--profile", action="store_true", help="per-kernel breakdown of one eager decode step instead of the sweep")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "generate_bench needs a GPU"
    print(json.dumps(card()), flush=True)
    if a.profile:
        for name in a.presets.split(","):
            profile_step(name, 8, 1024)
        return
    for name in a.presets.split(","):
        bench_preset(name, [int(x) for x in a.batches.split(",")], [int(x) for x in a.prompts.split(",")], a.new_tokens, a.window,
                     not a.no_hf)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
