"""GPU busy fraction inside one un-graphed training step (nsys is not in the image: torch.profiler's CUPTI activity
records give every kernel's start / end on the device, including the ctypes-launched ones of libodb200.so).

    python profiles/idle_gap.py [--graph]      -> profiles_out/idle_gap.json

Reports, for ONE optimizer step (16 micro-batches + AdamW) after warm-up: window (first kernel start -> last kernel end),
sum of kernel durations, busy %, number of kernels, and the distribution of the gaps between consecutive kernels.
"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from opendiloco_b200.models.config import LlamaConfig  # noqa: E402
from opendiloco_b200.models.llama import LlamaForCausalLM  # noqa: E402
from opendiloco_b200.trainer import DiLoCoTrainer, TrainerConfig  # noqa: E402

if "--graph" in sys.argv:
    os.environ["ODB_CUDA_GRAPH"] = "1"
dev = torch.device("cuda", 0)
cfg = LlamaConfig.from_pretrained("150m")
model = LlamaForCausalLM(cfg, device=dev, precision="bf16-mixed", seed=0)
tr = DiLoCoTrainer(model, TrainerConfig(grad_accum=16, local_steps=1000, samples_per_step=512))
ids = torch.randint(3, cfg.vocab_size, (32, 1024), device=dev)
batch = {"input_ids": ids, "labels": ids}


def it():
    while True:
        yield batch


g = it()
for _ in range(3):
    tr.train_step(g)
torch.cuda.synchronize()
from torch.profiler import ProfilerActivity, profile  # noqa: E402

with profile(activities=[ProfilerActivity.CUDA]) as prof:
    tr.train_step(g)
    torch.cuda.synchronize()
ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and e.time_range is not None]
spans = sorted((e.time_range.start, e.time_range.end, e.name) for e in ev if "memcpy" not in e.name.lower() or True)
t0, t1 = spans[0][0], max(s[1] for s in spans)
busy = 0.0
cur_s, cur_e = spans[0][0], spans[0][1]
gaps = []
for s, e, _ in spans[1:]:
    if s > cur_e:
        busy += cur_e - cur_s
        gaps.append(s - cur_e)
        cur_s, cur_e = s, e
    else:
        cur_e = max(cur_e, e)
busy += cur_e - cur_s
gaps.sort()
out = {"graph": "--graph" in sys.argv, "kernels": len(spans), "window_ms": (t1 - t0) / 1e3, "busy_ms": busy / 1e3,
       "busy_pct": 100.0 * busy / (t1 - t0), "idle_ms": (t1 - t0 - busy) / 1e3, "gaps": len(gaps),
       "gap_us_median": gaps[len(gaps) // 2] if gaps else 0, "gap_us_p90": gaps[int(len(gaps) * 0.9)] if gaps else 0,
       "gap_us_max": gaps[-1] if gaps else 0, "gaps_over_10us": sum(1 for x in gaps if x > 10)}
os.makedirs("profiles_out", exist_ok=True)
name = "profiles_out/idle_gap_graph.json" if out["graph"] else "profiles_out/idle_gap.json"
json.dump(out, open(name, "w"), indent=1)
print(json.dumps(out))
