"""One micro-batch (fwd+bwd) + optimizer step of Llama-150M between cudaProfilerStart/Stop, for
    ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv --log-file profiles_out/launches.csv python profiles/profile_step.py
(serialised, cold-cache: compare SHARES, not absolutes)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from opendiloco_b200 import DiLoCoTrainer, LlamaConfig, LlamaForCausalLM, TrainerConfig  # noqa: E402
from opendiloco_b200.utils.data import SyntheticTokenLoader  # noqa: E402

mb = int(os.environ.get("MB", 32))
model_name = os.environ.get("MODEL", "150m")
cfg = LlamaConfig.from_pretrained(model_name)
m = LlamaForCausalLM(cfg, device="cuda", seed=0)
tr = DiLoCoTrainer(m, TrainerConfig(grad_accum=1, local_steps=4, samples_per_step=mb))
ld = SyntheticTokenLoader(mb, 1024, vocab_size=cfg.vocab_size, seed=0, with_mask=False)
for _ in range(3):
    tr.train_step(ld)
torch.cuda.synchronize()
torch.cuda.profiler.start()
tr.train_step(ld)          # 4th step: includes the (solo) outer step
torch.cuda.synchronize()
torch.cuda.profiler.stop()
print("done")
