"""Per-kernel time of one eager optimizer step at the bench shape (Llama-150M, 16 micro-batches of 32 x 1024 tokens +
AdamW), from torch.profiler's CUDA activity records.

    python profiles/step_kernels.py [--root DIR]      -> profiles_out/step_kernels.json

--root DIR imports opendiloco_b200 from another built tree (e.g. an older commit).  Prints one line per kernel name:
total device time in the step, call count and share of the summed kernel time; the JSON holds the same rows."""
import argparse
import json
import os
import sys

os.environ["ODB_CUDA_GRAPH"] = "0"       # eager launches: every kernel is its own activity record
ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--out", default="profiles_out/step_kernels.json")
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from opendiloco_b200.models.config import LlamaConfig  # noqa: E402
from opendiloco_b200.models.llama import LlamaForCausalLM  # noqa: E402
from opendiloco_b200.trainer import DiLoCoTrainer, TrainerConfig  # noqa: E402

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
for _ in range(2):
    tr.train_step(g)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    tr.train_step(g)
    torch.cuda.synchronize()

rows = {}
for e in prof.events():
    if e.device_type != torch.autograd.DeviceType.CUDA or e.time_range is None:
        continue
    name = e.name.split("(")[0]            # without the parameter list: template arguments tell instantiations apart
    r = rows.setdefault(name, [0.0, 0])
    r[0] += e.time_range.end - e.time_range.start
    r[1] += 1
total = sum(r[0] for r in rows.values())
table = sorted(({"kernel": k, "total_us": v[0], "calls": v[1], "share": v[0] / total} for k, v in rows.items()),
               key=lambda r: -r["total_us"])
out = {"gpu": torch.cuda.get_device_name(dev), "root": os.path.abspath(args.root), "kernel_total_ms": total / 1e3,
       "kernels": table}
os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
json.dump(out, open(args.out, "w"), indent=1)
print(f"{out['gpu']}: summed kernel time of one optimizer step {total / 1e3:.1f} ms")
for r in table[:25]:
    print(f"{r['total_us'] / 1e3:9.2f} ms {r['calls']:6d} calls {100 * r['share']:5.1f} %  {r['kernel'][:110]}")
