"""High-level training API: the call a user (and ``bench.py``'s end-to-end arm) makes.

    trainer = DiLoCoTrainer(model, TrainerConfig(...), topology)
    for step in range(n):
        loss = trainer.train_step(loader)      # grad-accumulated inner step (+ outer step every local_steps)

One ``train_step`` = the body of the reference loops between two optimizer steps
(train_fsdp.py:361-413, train_diloco_torch.py:272-353): ``grad_accum`` micro-batches of forward/backward with the loss
divided by ``grad_accum``, worker-internal gradient reduction, global-norm clip, AdamW, LR schedule, zero-grad, and -
every ``local_steps`` steps - the DiLoCo outer step.  Host-side it issues: one pinned H2D copy per micro-batch, no
device->host read unless the caller asks for the loss value.
"""
from __future__ import annotations

from dataclasses import dataclass
from functools import partial
from typing import Iterator

import torch

from .models.llama import LlamaForCausalLM
from .optim.fused import FusedAdamW
from .optim.muon import FusedMuon
from .parallel import comm
from .parallel.diloco import AllReduceStrategy, DiLoCoOptimizer
from .parallel.swarm import DHT
from .utils.profiling import StepTimer, nvtx_range
from .utils.training import get_cosine_schedule_with_warmup


@dataclass
class TrainerConfig:
    lr: float = 4e-4
    weight_decay: float = 0.1
    betas: tuple = (0.9, 0.95)
    eps: float = 1e-8
    max_grad_norm: float = 1.0
    warmup_steps: int = 1000
    total_steps: int = 88_000
    grad_accum: int = 1
    # DiLoCo (None => plain data-parallel baseline, the reference's non-hv path)
    local_steps: int | None = 500
    outer_lr: float = 0.7
    outer_momentum: float = 0.9
    outer_nesterov: bool = True
    samples_per_step: int = 512          # per-worker batch (tracker bookkeeping: hivemind_diloco.py:395)
    sharding_strategy: str = "NO_SHARD"
    all_reduce_strategy: AllReduceStrategy = AllReduceStrategy.WAIT_FOR_ALL
    timeout_waiting_for_peers: float | None = None
    matchmaking_time: float | None = None
    averaging_timeout: float | None = None
    compression: object | None = None
    fused_collective: bool | None = None
    offload_device: str | None = None
    inner_optimizer: str = "adamw"       # "adamw" | "muon" (FusedMuon: Muon on the projection matrices, NO_SHARD only)
    muon_momentum: float = 0.95
    muon_adjust_lr_fn: str | None = "match_rms_adamw"


SHARDED = {"SHARD_GRAD_OP", "_HYBRID_SHARD_ZERO2", "FULL_SHARD", "HYBRID_SHARD"}


class DiLoCoTrainer:
    def __init__(self, model: LlamaForCausalLM, cfg: TrainerConfig, topo: comm.Topology | None = None):
        self.model, self.cfg = model, cfg
        if cfg.inner_optimizer not in ("adamw", "muon"):
            raise ValueError(f"unknown inner_optimizer {cfg.inner_optimizer!r}: choose 'adamw' or 'muon'")
        if cfg.inner_optimizer == "muon" and cfg.sharding_strategy in SHARDED:
            raise ValueError(f"inner_optimizer='muon' needs whole matrices: it supports NO_SHARD only, not {cfg.sharding_strategy}")
        self.topo = topo if topo is not None else comm.build_topology()
        shard = cfg.sharding_strategy in SHARDED
        inner_factory = partial(FusedAdamW, lr=cfg.lr, weight_decay=cfg.weight_decay, betas=cfg.betas, eps=cfg.eps,
                                max_grad_norm=cfg.max_grad_norm, zero_grad_in_step=True, dp_group=self.topo.inner_group,
                                shard=shard, shard_params=cfg.sharding_strategy in ("FULL_SHARD", "HYBRID_SHARD"))
        if cfg.inner_optimizer == "muon":
            inner_factory = partial(FusedMuon, lr=cfg.lr, weight_decay=cfg.weight_decay, momentum=cfg.muon_momentum,
                                    adjust_lr_fn=cfg.muon_adjust_lr_fn, adamw_betas=cfg.betas, adamw_eps=cfg.eps,
                                    max_grad_norm=cfg.max_grad_norm, zero_grad_in_step=True, dp_group=self.topo.inner_group)
        sched_factory = partial(get_cosine_schedule_with_warmup, num_warmup_steps=cfg.warmup_steps,
                                num_training_steps=cfg.total_steps)
        params = list(model.parameters())
        if cfg.local_steps is not None:
            self.dht = DHT(start=True, group=self.topo.outer_group) if self.topo.outer_group is not None else None
            kw = {}
            if cfg.matchmaking_time is not None:
                kw["matchmaking_time"] = cfg.matchmaking_time
            if cfg.averaging_timeout is not None:
                kw["averaging_timeout"] = cfg.averaging_timeout
            self.optimizer = DiLoCoOptimizer(
                dht=self.dht, run_id="llama", batch_size=cfg.samples_per_step, num_inner_steps=cfg.local_steps,
                outer_optimizer=partial(torch.optim.SGD, lr=cfg.outer_lr, momentum=cfg.outer_momentum,
                                        nesterov=cfg.outer_nesterov),
                inner_optimizer=inner_factory, params=params, scheduler=None,
                all_reduce_strategy=cfg.all_reduce_strategy, timeout_waiting_for_peers=cfg.timeout_waiting_for_peers,
                grad_compression=cfg.compression, fused_collective=cfg.fused_collective,
                offload_device=cfg.offload_device, **kw)
            self.inner = self.optimizer.inner_optimizer
        else:
            self.dht = None
            self.optimizer = inner_factory(params)
            self.inner = self.optimizer
        self.scheduler = sched_factory(self.inner)
        self.real_step = 0
        self.device = model.device
        self._loss_acc = torch.zeros((), dtype=torch.float32, device=self.device)
        self.timer = StepTimer(enabled=False)        # trainer.timer.enabled = True to collect inner/outer CUDA-event timings

    # ------------------------------------------------------------------------------------------------
    @property
    def is_diloco(self) -> bool:
        return isinstance(self.optimizer, DiLoCoOptimizer)

    def broadcast_initial_weights(self) -> None:
        """All workers start from rank-0 weights: ONE flat broadcast (reference N1: 111 broadcasts,
        train_diloco_torch.py:253-255)."""
        import torch.distributed as dist

        if dist.is_initialized() and dist.get_world_size() > 1:
            dist.broadcast(self.model.arena.master, src=0)
            self.model.arena.sync_shadow()
            if self.is_diloco:
                sa = self.optimizer.state_averager
                sa.theta_outer.copy_(sa.theta_local)

    def micro_step(self, batch: dict, loss_scale: float) -> torch.Tensor:
        dev = self.device
        ids = batch["input_ids"].to(dev, non_blocking=True)
        lab = batch["labels"]
        labels = ids if lab is batch["input_ids"] else lab.to(dev, non_blocking=True)
        return self.model.forward_backward(ids, labels, loss_scale, batch.get("attention_mask_device"))

    def train_step(self, batches: Iterator[dict]) -> torch.Tensor:
        """Run one optimizer step, pulling ``grad_accum`` micro-batches from ``batches``.  Returns the summed
        (already 1/grad_accum-scaled) loss as a device scalar, like the reference's ``loss_batch``."""
        cfg = self.cfg
        self._loss_acc.zero_()
        scale = 1.0 / cfg.grad_accum
        self.timer.start("inner_step")
        with nvtx_range("micro_batches"):
            for _ in range(cfg.grad_accum):
                loss = self.micro_step(next(batches), scale)
                self._loss_acc.add_(loss, alpha=scale)
        with nvtx_range("optimizer_step"):
            self.optimizer.step()      # clip + AdamW (+ outer step when due); gradients zeroed by the fused kernel
        self.timer.stop("inner_step")
        self.scheduler.step()
        self.real_step += 1
        return self._loss_acc

    def lr(self) -> float:
        return self.inner.param_groups[0]["lr"]
