"""Reference arm of bench.py: runs the UNMODIFIED reference (``baseline/_ref/open_diloco/train_diloco_torch.py``, installed
with ``pip --target baseline/_ref --no-deps /tmp/<copy of /root/reference>``) through its own ``main(**flags)`` entry
point and stock code path (HF LlamaForCausalLM, torch.autocast, torch AdamW/SGD, per-parameter NCCL all_reduce, CPU
offload of the outer parameters).

Nothing in ``baseline/_ref`` is edited.  What the offline box lacks is provided from OUTSIDE the reference:
  * ``cyclopts`` (not installed): a 10-line stand-in so ``@app.default`` decorates ``main``;
  * ``get_grad_norm`` / ``register_hooks_log_activations``: the reference HEAD imports these two names from
    ``open_diloco.utils`` although that module does not define them (SURVEY.md §0 "latent breakage"); they are only
    called when ``--log-activations-steps`` is set, so inert placeholders are attached before the import;
  * the Mistral tokenizer and the C4 stream need the network: ``AutoTokenizer.from_pretrained`` returns a locally built
    ``PreTrainedTokenizerFast`` (same pad = "</s>" = id 2) and ``load_dataset`` returns a synthetic pre-tokenised
    stream - the same token law our arm uses.  HF's real ``DataCollatorForLanguageModeling`` and torch ``DataLoader``
    still do the batching;
  * the model directory is a random-init Llama-150M saved with ``save_pretrained`` (hub checkpoints are unreachable);
  * wandb runs with ``WANDB_MODE=disabled``.
Timing brackets exactly K optimizer steps from inside the data stream (barrier + synchronize on both sides).
"""
from __future__ import annotations

import json
import os
import sys
import tempfile
import time
import types

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _install_shims():
    if "cyclopts" not in sys.modules:
        m = types.ModuleType("cyclopts")

        class App:
            def default(self, fn):
                self._fn = fn
                return fn

            def __call__(self, *a, **k):
                return self._fn(*a, **k)

        m.App = App
        sys.modules["cyclopts"] = m
    os.environ.setdefault("WANDB_MODE", "disabled")
    os.environ.setdefault("WANDB_SILENT", "true")
    os.environ.setdefault("TOKENIZERS_PARALLELISM", "false")
    os.environ.setdefault("HF_HUB_OFFLINE", "1")
    sys.path.insert(0, os.path.join(HERE, "_ref"))
    import open_diloco.utils as u   # the reference's own module

    if not hasattr(u, "get_grad_norm"):
        u.get_grad_norm = lambda model: {}
    if not hasattr(u, "register_hooks_log_activations"):
        u.register_hooks_log_activations = lambda model: ([], {})


def _local_tokenizer(vocab_size: int):
    from tokenizers import Tokenizer, models
    from transformers import PreTrainedTokenizerFast

    vocab = {"<unk>": 0, "<s>": 1, "</s>": 2}
    for i in range(3, vocab_size):
        vocab[f"t{i}"] = i
    tok = Tokenizer(models.WordLevel(vocab, unk_token="<unk>"))
    return PreTrainedTokenizerFast(tokenizer_object=tok, unk_token="<unk>", bos_token="<s>", eos_token="</s>", pad_token="</s>")


def run(a, ClockSampler) -> dict:
    import torch
    import torch.distributed as dist

    _install_shims()
    import open_diloco.train_diloco_torch as ref

    world = int(os.environ.get("WORLD_SIZE", 1))
    rank = int(os.environ.get("RANK", 0))
    local_rank = int(os.environ.get("LOCAL_RANK", 0))
    os.environ.setdefault("LOCAL_RANK", "0")
    os.environ.setdefault("RANK", "0")
    os.environ.setdefault("WORLD_SIZE", "1")
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29533")
    assert world == a.gpus, f"--gpus {a.gpus} but WORLD_SIZE={world}"
    ref.ddp_setup()                                   # reference: init_process_group("nccl") + set_device

    cfg_json = json.load(open(os.path.join(ROOT, "opendiloco_b200", "configs", f"config_{a.model}.json")))
    vocab = cfg_json.get("vocab_size", 32000)
    accum = a.batch // a.micro_batch
    H = a.local_steps if a.local_steps is not None else a.warmup + a.steps
    total_steps = a.warmup + a.steps
    samples_total = total_steps * a.batch
    timed_from = a.warmup * a.batch

    # -- random-init checkpoint directory (rank 0 writes, everyone loads)
    model_dir = os.path.join(tempfile.gettempdir(), f"odb_ref_llama_{a.model}")
    if rank == 0 and not os.path.exists(os.path.join(model_dir, "config.json")):
        from transformers import LlamaConfig, LlamaForCausalLM

        torch.manual_seed(0)
        hf_cfg = LlamaConfig(**{k: v for k, v in cfg_json.items() if k not in ("architectures", "model_type")})
        LlamaForCausalLM(hf_cfg).save_pretrained(model_dir)
    dist.barrier(device_ids=[local_rank])

    marks = {}

    def sync():
        torch.cuda.synchronize()
        dist.barrier(device_ids=[local_rank])
        torch.cuda.synchronize()

    sampler = ClockSampler(local_rank)

    class Stream(torch.utils.data.IterableDataset):
        def __iter__(self):
            gen = torch.Generator().manual_seed(1234 * 1_000_003 + rank)
            mask = [1] * a.seq
            for i in range(samples_total):
                if i == timed_from:
                    sync()
                    sampler.start()
                    marks["t0"] = time.perf_counter()
                yield {"input_ids": torch.randint(3, vocab, (a.seq,), generator=gen).tolist(), "attention_mask": mask}
            sync()
            marks["t1"] = time.perf_counter()
            marks["clocks"] = sampler.stop()

    class FakeDatasetDict(dict):
        def map(self, *args, **kwargs):
            return self

        def shuffle(self, *args, **kwargs):
            return self

    ref.load_dataset = lambda *args, **kwargs: FakeDatasetDict(train=Stream(), validation=Stream())
    ref.split_dataset_by_node = lambda ds, world_size, rank: ds

    class _Tok:
        @staticmethod
        def from_pretrained(*args, **kwargs):
            return _local_tokenizer(vocab)

    ref.AutoTokenizer = _Tok

    ckpt_dir = os.path.join(tempfile.gettempdir(), "odb_ref_outputs")
    ref.main(batch_size=a.batch, per_device_train_batch_size=a.micro_batch, seq_length=a.seq, checkpoint_path=ckpt_dir,
             warmup_steps=1000, total_steps=88_000, precision="bf16-mixed", project="odb_bench_reference",
             model_name_or_path=model_dir, lr=4e-4, local_steps=H, outer_lr=0.7)

    elapsed = torch.tensor([marks["t1"] - marks["t0"]], dtype=torch.float64, device=f"cuda:{local_rank}")
    dist.all_reduce(elapsed, op=dist.ReduceOp.MAX)
    secs = float(elapsed.item())
    tokens_per_step = a.batch * a.seq * world
    value = tokens_per_step * a.steps / secs
    out = {
        "metric": "tokens_per_sec (DiLoCo inner steps incl. one outer sync in the timed window)",
        "value": value, "unit": "tokens/s", "n_gpus": world, "steps": a.steps, "warmup": a.warmup,
        "ms_per_step": secs * 1e3 / a.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "bf16", "data": "synthetic tokens (uniform over vocab), random-init weights", "impl": "reference",
        "config": {"model": f"llama-{a.model}", "global_batch": a.batch * world, "per_worker_batch": a.batch,
                   "micro_batch": a.micro_batch, "grad_accum": accum, "seq_len": a.seq, "parallelism": f"diloco{world}x1",
                   "local_steps": H, "outer_steps_in_timed_window": 1 if H <= total_steps and H > a.warmup else 0},
        "notes": {"entry": "open_diloco.train_diloco_torch.main (unmodified, baseline/_ref)", "l2": "per-step working set >> 50 MB L2",
                  "inner_opt": "AdamW lr4e-4 wd0.1 b(0.9,0.95) clip1.0 cosine(1000,88000)", "outer_opt": "SGD lr0.7 m0.9 nesterov"},
        "tokens_per_sec_per_gpu": value / world,
        "clocks": marks.get("clocks"),
        "e2e": {"value": value, "unit": "tokens/s", "h2d_bytes_per_step": a.micro_batch * a.seq * 8 * 3 * accum,
                "d2h_bytes_per_step": 4,
                "note": "the reference's stock loop is inherently end-to-end (pageable H2D of ids/mask/labels every "
                        "micro-batch, loss .item() every step on rank 0); wall-clock between barriers"},
        "gpu_launches": None,
    }
    ref.destroy_process_group()
    return out if rank == 0 else {}
