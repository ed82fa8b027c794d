"""Loss-curve parity on the GPU/bf16 path: the UNMODIFIED reference loop (baseline/_ref train_diloco_torch.py: HF Llama under
torch.autocast(bf16), torch AdamW / cosine schedule / clip / SGD-Nesterov outer step) against this framework's kernels, on
IDENTICAL initial weights (one random-init HF checkpoint), an IDENTICAL token stream (torch.Generator seeded per step) and
identical hyper-parameters.  BASELINE.md asks for |d loss| <= 1e-3 at step 1000.

    python profiles/loss_parity.py --impl reference --steps 1000 --out profiles_out/parity_ref.jsonl
    python profiles/loss_parity.py --impl ours      --steps 1000 --out profiles_out/parity_ours.jsonl
    python profiles/loss_parity.py --compare profiles_out/parity_ref.jsonl profiles_out/parity_ours.jsonl

Protocol: Llama-150M, 1 worker (the outer step is the solo form), 32 x 1024 tokens per optimizer step (one micro-batch),
H = 50, lr 4e-4 with 100 warm-up steps of a 1000-step cosine, bf16-mixed.  (The full 512 x 1024 batch would cost the
reference arm ~35 GPU-minutes for 1000 steps.)
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "baseline"))

ap = argparse.ArgumentParser()
ap.add_argument("--impl", choices=["ours", "reference"], default="ours")
ap.add_argument("--steps", type=int, default=1000)
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--seq", type=int, default=1024)
ap.add_argument("--local-steps", type=int, default=50)
ap.add_argument("--warmup", type=int, default=100)
ap.add_argument("--model", default="150m")
ap.add_argument("--out", default="profiles_out/parity.jsonl")
ap.add_argument("--compare", nargs=2)
a = ap.parse_args()

if a.compare:
    load = lambda p: {json.loads(l)["step"]: json.loads(l)["loss"] for l in open(p) if l.strip()}   # noqa: E731
    r, o = load(a.compare[0]), load(a.compare[1])
    steps = sorted(set(r) & set(o))
    worst = max(abs(r[s] - o[s]) for s in steps)
    print(f"common steps: {len(steps)}   worst |d loss| over the run: {worst:.4e}")
    for s in (1, 10, 50, 100, 200, 500, 1000):
        if s in r and s in o:
            print(f"step {s:5d}: reference {r[s]:.5f}   ours {o[s]:.5f}   |d| {abs(r[s] - o[s]):.2e}")
    win = [s for s in steps if s > max(steps) - 20]
    print(f"mean over the last 20 steps: reference {sum(r[s] for s in win) / len(win):.5f}   ours {sum(o[s] for s in win) / len(win):.5f}")
    sys.exit(0)

import torch  # noqa: E402

os.environ.setdefault("LOCAL_RANK", "0"); os.environ.setdefault("RANK", "0"); os.environ.setdefault("WORLD_SIZE", "1")  # noqa: E702
os.environ.setdefault("MASTER_ADDR", "127.0.0.1"); os.environ.setdefault("MASTER_PORT", "29541")  # noqa: E702
from run_reference_fsdp import make_model_dir  # noqa: E402

model_dir, vocab = make_model_dir(a.model, 0)


def tokens_for_step(step: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(777_000 + step)
    return torch.randint(3, vocab, (a.batch, a.seq), generator=g)


os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
out = open(a.out, "w")

if a.impl == "reference":
    import run_reference as rr

    rr._install_shims()
    import open_diloco.train_diloco_torch as ref

    ref.ddp_setup()

    class Stream(torch.utils.data.IterableDataset):
        def __iter__(self):
            mask = [1] * a.seq
            for s in range(1, a.steps + 1):
                for row in tokens_for_step(s).tolist():
                    yield {"input_ids": row, "attention_mask": mask}

    class FakeDatasetDict(dict):
        def map(self, *args, **kwargs):
            return self

        def shuffle(self, *args, **kwargs):
            return self

    ref.load_dataset = lambda *args, **kwargs: FakeDatasetDict(train=Stream(), validation=Stream())
    ref.split_dataset_by_node = lambda ds, world_size, rank: ds
    ref.AutoTokenizer = type("_Tok", (), {"from_pretrained": staticmethod(lambda *x, **k: rr._local_tokenizer(vocab))})
    capture = lambda d, *x, **k: (out.write(json.dumps({"step": int(d["step"]), "loss": float(d["Loss"])}) + "\n"), out.flush())  # noqa: E731
    stock_init = ref.wandb.init

    def init_then_capture(*x, **k):        # wandb.init() re-binds wandb.log to the run's method: install the tap afterwards
        r = stock_init(*x, **k)
        ref.wandb.log = capture
        return r

    ref.wandb.init = init_then_capture
    ref.main(batch_size=a.batch, per_device_train_batch_size=a.batch, seq_length=a.seq, checkpoint_path="/tmp/odb_parity_ckpt",
             warmup_steps=a.warmup, total_steps=a.steps, precision="bf16-mixed", project="odb_parity", model_name_or_path=model_dir,
             lr=4e-4, local_steps=a.local_steps, outer_lr=0.7)
else:
    from opendiloco_b200.models.llama import LlamaForCausalLM
    from opendiloco_b200.trainer import DiLoCoTrainer, TrainerConfig

    dev = torch.device("cuda", 0)
    model = LlamaForCausalLM.from_pretrained(model_dir, device=dev, precision="bf16-mixed")
    tr = DiLoCoTrainer(model, TrainerConfig(grad_accum=1, local_steps=a.local_steps, samples_per_step=a.batch, warmup_steps=a.warmup,
                                            total_steps=a.steps, lr=4e-4))

    def batches():
        s = 0
        while True:
            s += 1
            ids = tokens_for_step(s).pin_memory()
            yield {"input_ids": ids, "labels": ids}

    it = batches()
    for s in range(1, a.steps + 1):
        loss = float(tr.train_step(it).item())
        out.write(json.dumps({"step": s, "loss": loss}) + "\n")
    out.flush()
out.close()
print(f"wrote {a.out}")
