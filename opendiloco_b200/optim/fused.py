"""Single-launch optimizers over a flat parameter buffer, with optional ZeRO sharding inside a DiLoCo worker.

``FusedAdamW``   - inner optimizer (reference: torch.optim.AdamW(lr, weight_decay=0.1, betas=(0.9,0.95)) at
                   train_fsdp.py:250 / train_diloco_torch.py:186) with global-norm clipping, bf16 shadow refresh and
                   (optionally) gradient zeroing folded into the same kernel (SURVEY.md §2.5 K9-K12).
                   With ``dp_group`` it is also the worker-internal data parallelism:
                     * ``shard=False`` (NO_SHARD): one flat gradient all-reduce (reference N3: FSDP NO_SHARD)
                     * ``shard=True``  (SHARD_GRAD_OP / _HYBRID_SHARD_ZERO2): flat reduce-scatter of gradients, AdamW on
                       the rank's slice of (master, m, v), all-gather of the bf16 compute weights (reference N4).
                     * ``shard_params=True`` (FULL_SHARD / HYBRID_SHARD) additionally keeps the compute weights sharded
                       between uses: the engine all-gathers them before forward and again before backward and frees the
                       gathered copy after each (FSDP's reshard_after_forward on the reference's single flat unit).
``flatten_params`` re-homes arbitrary ``nn.Parameter``s into one contiguous fp32 buffer so every model, not only
                   the arena-backed Llama, gets the flat fast path.

torch-compatible ``state_dict()`` layouts are kept (per-parameter ``exp_avg``/``exp_avg_sq``/``step`` views into the
flat moment buffers; a single flat entry when sharded) so reference-style checkpoint code round-trips them.
"""
from __future__ import annotations

import weakref
from typing import Iterable

import torch
import torch.distributed as dist

from ..ops import kernels as K


class FlatView:
    """Parameters that are consecutive views of one flat fp32 buffer (+ matching flat grad buffer).

    ``lo:hi`` is the slice this rank's optimizers own (the whole buffer unless ZeRO-sharded)."""

    def __init__(self, params: list[torch.nn.Parameter], flat: torch.Tensor, grad: torch.Tensor, offsets: list[int],
                 shadow: torch.Tensor | None = None):
        self.params, self.flat, self.grad, self.offsets, self.shadow = params, flat, grad, offsets, shadow
        self.lo, self.hi = 0, flat.numel()
        self.shard_group = None
        self.param_sharded = False           # FULL_SHARD: compute weights kept as per-rank shards between uses
        self.arena = getattr(params[0], "_odb_arena", None) if params else None

    @property
    def numel(self) -> int:
        return self.flat.numel()

    @property
    def sharded(self) -> bool:
        return self.shard_group is not None

    def set_shard(self, group) -> None:
        n, r = dist.get_world_size(group), dist.get_rank(group)
        assert self.flat.numel() % (n * 4) == 0
        per = self.flat.numel() // n
        self.lo, self.hi, self.shard_group = r * per, (r + 1) * per, group

    def own(self, buf: torch.Tensor | None) -> torch.Tensor | None:
        return None if buf is None else buf[self.lo:self.hi]

    def own_shadow(self) -> torch.Tensor | None:
        """This rank's slice of the low-precision compute weights (the persistent shard under FULL_SHARD)."""
        if self.param_sharded:
            return self.arena.shadow_shard
        return self.own(self.shadow)

    def shard_parameters(self) -> None:
        """FULL_SHARD / HYBRID_SHARD on top of set_shard(): the gathered compute weights are released between uses."""
        if self.arena is None or self.shadow is None or not self.sharded:
            return
        self.arena.enable_param_sharding(self.shard_group, self.lo, self.hi)
        self.param_sharded = self.arena.param_sharded
        if self.param_sharded:
            self.shadow = None

    def view_of(self, buf: torch.Tensor, i: int) -> torch.Tensor:
        p = self.params[i]
        return buf[self.offsets[i]:self.offsets[i] + p.numel()].view(p.shape)

    @torch.no_grad()
    def rehome(self, new_flat: torch.Tensor) -> None:
        """Move the fp32 master weights into ``new_flat`` (e.g. an NVLink symmetric-memory allocation) and re-point every
        parameter view at it.  Values are preserved; optimizer moments / gradients are separate buffers and stay."""
        assert new_flat.numel() == self.flat.numel() and new_flat.dtype == self.flat.dtype and new_flat.device == self.flat.device
        new_flat.copy_(self.flat)
        fp32_compute = self.shadow is None and not self.param_sharded
        if self.arena is not None:
            self.arena.adopt_master(new_flat)
        self.flat = new_flat
        for p, o in zip(self.params, self.offsets):
            p.data = new_flat[o:o + p.numel()].view(p.shape)
        assert fp32_compute == (self.shadow is None and not self.param_sharded)

    @torch.no_grad()
    def rehome_grad(self, new_grad: torch.Tensor) -> None:
        """Move the fp32 gradient accumulator into ``new_grad`` (a symmetric-memory window) and re-point ``p.grad``."""
        assert new_grad.numel() == self.grad.numel() and new_grad.dtype == self.grad.dtype
        new_grad.copy_(self.grad)
        if self.arena is not None:
            self.arena.grad = new_grad
            self.arena.version += 1
        self.grad = new_grad
        for p, o in zip(self.params, self.offsets):
            p.grad = new_grad[o:o + p.numel()].view(p.shape)

    @torch.no_grad()
    def rehome_shadow(self, new_shadow: torch.Tensor) -> None:
        assert self.shadow is not None and new_shadow.numel() == self.shadow.numel() and new_shadow.dtype == self.shadow.dtype
        new_shadow.copy_(self.shadow)
        if self.arena is not None:
            self.arena.shadow = new_shadow
            self.arena.version += 1
        self.shadow = new_shadow

    @torch.no_grad()
    def gather_compute_weights(self) -> None:
        """After a sharded update: every rank publishes its slice of the compute weights (bf16 shadow, or fp32 master
        when computing in fp32) to the worker's other GPUs."""
        if not self.sharded or self.param_sharded:      # FULL_SHARD gathers at the start of forward / backward instead
            return
        buf = self.shadow if self.shadow is not None else self.flat
        dist.all_gather_into_tensor(buf, buf[self.lo:self.hi], group=self.shard_group)


def flatten_params(params: Iterable[torch.nn.Parameter]) -> FlatView:
    """Return a FlatView over ``params``; arena-backed parameters are used in place, others are re-homed."""
    params = list(params)
    assert params, "no parameters"
    arena = getattr(params[0], "_odb_arena", None)
    if arena is not None and all(getattr(p, "_odb_arena", None) is arena for p in params):
        offs = [arena.slots[p._odb_name].offset for p in params]
        shadow = arena.shadow if arena.shadow is not arena.master else None
        return FlatView(params, arena.master, arena.grad, offs, shadow)
    dev = params[0].device
    assert all(p.device == dev and p.dtype == torch.float32 for p in params), "flat optimizers need fp32 params on one device"
    offs, off = [], 0
    for p in params:
        off = (off + 31) // 32 * 32
        offs.append(off)
        off += p.numel()
    total = (off + 1023) // 1024 * 1024
    flat = torch.zeros(total, dtype=torch.float32, device=dev)
    grad = torch.zeros(total, dtype=torch.float32, device=dev)
    for p, o in zip(params, offs):
        flat[o:o + p.numel()].copy_(p.data.reshape(-1))
        if p.grad is not None:
            grad[o:o + p.numel()].copy_(p.grad.reshape(-1))
        p.data = flat[o:o + p.numel()].view(p.shape)
        p.grad = grad[o:o + p.numel()].view(p.shape)
    return FlatView(params, flat, grad, offs, None)


class FusedAdamW(torch.optim.Optimizer):
    """AdamW with decoupled weight decay over a flat buffer; one kernel per step (plus one norm pass when clipping).

    ``max_grad_norm`` folds ``clip_grad_norm_`` into the step; an external ``model.clip_grad_norm_(1.0)`` call
    (reference loop order: clip, then step) hands its partial norms to the next step instead of rescaling gradients.
    """

    HP_RING = 8

    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-2,
                 max_grad_norm: float | None = None, zero_grad_in_step: bool = False, dp_group=None, shard: bool = False,
                 shard_params: bool = False):
        params = list(params)
        if params and isinstance(params[0], dict):
            assert len(params) == 1, "FusedAdamW supports a single param group (the reference uses one)"
            group_over = {k: v for k, v in params[0].items() if k != "params"}
            params = list(params[0]["params"])
        else:
            group_over = {}
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay)
        self.fv = flatten_params(params)
        super().__init__([{"params": params, **group_over}], defaults)
        self.dp_group = dp_group if (dp_group is not None and dist.get_world_size(dp_group) > 1) else None
        if self.dp_group is not None and shard:
            self.fv.set_shard(self.dp_group)
            if shard_params:
                self.fv.shard_parameters()
        fv = self.fv
        dev = fv.flat.device
        self.exp_avg = torch.zeros(fv.hi - fv.lo, dtype=torch.float32, device=dev)
        self.exp_avg_sq = torch.zeros(fv.hi - fv.lo, dtype=torch.float32, device=dev)
        self.max_grad_norm = max_grad_norm
        self.zero_grad_in_step = zero_grad_in_step
        self._step = 0                                                # step() calls, skipped ones included
        # steps a non-finite gradient skipped so far, counted by the step kernels themselves (two slots, see
        # adamw_bias_corrections in csrc/common.cuh): the bias corrections follow the updates actually applied, as torch's
        # AdamW under a GradScaler does, without the host ever reading the verdict
        self._skipped = torch.zeros(2, dtype=torch.int32, device=dev)
        # per-step scalars travel through a RING of pinned slots, each guarded by an event recorded after its H2D copy: the
        # host may run ahead of the GPU by several steps (only rank 0 reads the loss), and a single slot would be
        # rewritten before the asynchronous copy of an earlier step has read it
        self._hp_ring = [torch.zeros(K.HP_SIZE, dtype=torch.float32, pin_memory=dev.type == "cuda") for _ in range(self.HP_RING)]
        self._hp_events: list = [None] * self.HP_RING
        self._hp_slot = 0
        self._hp = torch.zeros(K.HP_SIZE, dtype=torch.float32, device=dev)
        self._partials = torch.zeros(K.MAX_PARTIALS, dtype=torch.float32, device=dev)
        self._flag = torch.zeros(1, dtype=torch.int32, device=dev)
        self.stats = torch.zeros(2, dtype=torch.float32, device=dev)   # [grad_norm, clip_coef] of the last step
        self._pending: tuple[int, float] | None = None                # (n_partials, max_norm) from clip_grad_norm_
        self._grads_synced = False
        self._inv_scale: torch.Tensor | None = None                   # 1/loss-scale handed over by unscale_()
        arena = getattr(params[0], "_odb_arena", None)
        if arena is not None:
            arena.fused_optimizer = weakref.ref(self)                 # lets model.clip_grad_norm_() find us
        self._init_state_views()
        # ZeRO-sharded worker on NVLink: reduce-scatter + clip + AdamW + all-gather as ONE kernel (csrc/zero_comm.cu)
        self._zero = None
        if self.dp_group is not None and self.fv.sharded and dev.type == "cuda":
            from .zero_fused import FusedZeroStep

            self._zero = FusedZeroStep.try_create(self)

    # ----------------------------------------------------------------- torch-compatible per-param state
    def _init_state_views(self) -> None:
        fv = self.fv
        if fv.sharded:
            # parameter boundaries do not align with shard boundaries: expose the shard as one flat entry on param 0
            self.state[fv.params[0]] = {"step": torch.tensor(float(self._step)), "exp_avg": self.exp_avg,
                                        "exp_avg_sq": self.exp_avg_sq, "shard": torch.tensor([fv.lo, fv.hi])}
            return
        for i, p in enumerate(fv.params):
            self.state[p] = {"step": torch.tensor(float(self._step)), "exp_avg": fv.view_of(self.exp_avg, i),
                             "exp_avg_sq": fv.view_of(self.exp_avg_sq, i)}

    def applied_steps(self) -> int:
        """Updates actually applied (torch's ``state["step"]``): step() calls minus the skipped ones.  Reads the device."""
        return self._step - int(self._skipped[(self._step + 1) & 1])

    def restore_step_count(self, step: int) -> None:
        """Continue from ``step`` applied updates (a checkpoint's count)."""
        self._step = step
        self._skipped.zero_()

    def state_dict(self):
        step = self.applied_steps()
        for st in self.state.values():
            st["step"] = torch.tensor(float(step))
        return super().state_dict()

    def load_state_dict(self, state_dict) -> None:
        super().load_state_dict(state_dict)
        # torch replaced our views with copies: pull the values back into the flat buffers and re-point
        fv, step = self.fv, 0
        if fv.sharded:
            st = self.state.get(fv.params[0], {})
            if "exp_avg" in st:
                self.exp_avg.copy_(st["exp_avg"].reshape(-1))
                self.exp_avg_sq.copy_(st["exp_avg_sq"].reshape(-1))
                step = int(float(st.get("step", 0)))
        else:
            for i, p in enumerate(fv.params):
                st = self.state.get(p, {})
                if "exp_avg" in st:
                    fv.view_of(self.exp_avg, i).copy_(st["exp_avg"])
                    fv.view_of(self.exp_avg_sq, i).copy_(st["exp_avg_sq"])
                    step = int(float(st.get("step", 0)))
        self.restore_step_count(step)
        self.state.clear()
        self._init_state_views()

    # ----------------------------------------------------------------- gradient synchronisation inside the worker
    @torch.no_grad()
    def sync_grads(self) -> None:
        """Average gradients over the worker's GPUs: flat all-reduce (NO_SHARD) or in-place flat reduce-scatter
        (ZeRO-2).  Idempotent per step; called by clip_grad_norm_ or step(), whichever comes first."""
        if self.dp_group is None or self._grads_synced or self._zero is not None:   # fused ZeRO: reduced inside the step kernel
            return
        fv = self.fv
        if fv.sharded:
            if fv.grad.is_cuda:
                dist.reduce_scatter_tensor(fv.grad[fv.lo:fv.hi], fv.grad, op=dist.ReduceOp.AVG, group=self.dp_group)
            else:
                dist.all_reduce(fv.grad, op=dist.ReduceOp.SUM, group=self.dp_group)
                fv.grad.div_(dist.get_world_size(self.dp_group))
        else:
            if fv.grad.is_cuda:
                dist.all_reduce(fv.grad, op=dist.ReduceOp.AVG, group=self.dp_group)
            else:
                dist.all_reduce(fv.grad, op=dist.ReduceOp.SUM, group=self.dp_group)
                fv.grad.div_(dist.get_world_size(self.dp_group))
        self._grads_synced = True

    # ----------------------------------------------------------------- clipping hand-off
    @torch.no_grad()
    def _norm_partials(self) -> int:
        """One pass over this rank's gradients: per-CTA sums of squares + the non-finite flag (K9 / K11)."""
        fv = self.fv
        self._flag.zero_()
        n = K.grad_sqnorm(fv.own(fv.grad), self._partials, self._flag)
        if fv.sharded:   # every shard has the same size => the same number of partials: sum them element-wise
            dist.all_reduce(self._partials[:n], op=dist.ReduceOp.SUM, group=self.dp_group)
            dist.all_reduce(self._flag, op=dist.ReduceOp.MAX, group=self.dp_group)   # an overflow anywhere skips everywhere
        return n

    @torch.no_grad()
    def compute_grad_norm_partials(self, max_norm: float) -> torch.Tensor:
        """Launch the norm pass now and remember it for the next step(); returns the (device) total norm lazily.
        Under a GradScaler the returned norm is that of the still-scaled gradients times 1/scale."""
        if self._zero is not None:
            # the fused ZeRO kernel reduces, measures and clips in one launch: only remember the threshold.  The returned
            # tensor is the norm slot that launch fills (it holds the previous step's norm until then).
            self._pending = (-1, float(max_norm))
            return self.stats[0]
        self.sync_grads()
        n = self._norm_partials()
        self._pending = (n, float(max_norm))
        total = self._partials[:n].sum().sqrt()
        if self._inv_scale is not None:
            total = total * self._inv_scale
        return total

    # ----------------------------------------------------------------- GradScaler (fp16-mixed) on the kernel path
    @torch.no_grad()
    def unscale_(self, scaler) -> None:
        """Stand-in for ``scaler.unscale_(optimizer)`` (train_fsdp.py:391-393): nothing is rescaled in memory - 1/scale
        becomes the ``grad_scale_inv`` hyper-parameter of the fused step (K11 folded into K9/K10), and the non-finite
        check is the flag of the norm pass, taken AFTER the worker-internal gradient reduction so every GPU of a worker
        sees the same verdict."""
        if not scaler.is_enabled():
            return
        if scaler._scale is None:
            scaler._lazy_init_scale_growth_tracker(self.fv.flat.device)
        self._inv_scale = scaler._scale.to(self.fv.flat.device, torch.float32).reciprocal()

    @torch.no_grad()
    def step_scaled(self, scaler):
        """``scaler.step(optimizer)`` on the kernel path: unscale + inf-check + clip + AdamW in the fused launches; the
        verdict is handed to the scaler so ``scaler.update()`` / ``found_inf_grad`` (utils.py:124-135) work unchanged."""
        if not scaler.is_enabled():
            return self.step()
        from torch.amp.grad_scaler import OptState

        if self._inv_scale is None:
            self.unscale_(scaler)
        self.step(_check_inf=True)
        st = scaler._per_optimizer_states[id(self)]
        st["found_inf_per_device"] = {self._flag.device: self._flag.to(torch.float32)}
        st["stage"] = OptState.STEPPED
        return None

    # ----------------------------------------------------------------- step
    def _upload_hp(self, values: dict) -> None:
        slot = self._hp_slot
        self._hp_slot = (slot + 1) % self.HP_RING
        ev = self._hp_events[slot]
        if ev is not None:
            ev.synchronize()                      # the copy that last read this slot has finished (normally long ago)
        hp = self._hp_ring[slot]
        for k, v in values.items():
            hp[k] = v
        self._hp.copy_(hp, non_blocking=True)
        if self._hp.is_cuda:
            ev = ev or torch.cuda.Event()
            ev.record(torch.cuda.current_stream(self._hp.device))
            self._hp_events[slot] = ev

    @torch.no_grad()
    def step(self, closure=None, _check_inf: bool = False):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self.sync_grads()
        fv = self.fv
        g = self.param_groups[0]
        self._step += 1
        max_norm = self.max_grad_norm
        n_part = 0
        if self._pending is not None:
            n_part, max_norm = self._pending
            self._pending = None
        elif self._zero is not None:
            n_part = -1
        elif (max_norm is not None and max_norm > 0) or _check_inf:
            n_part = self._norm_partials()
        self._upload_hp(K.adamw_hp(g["lr"], g["betas"], g["eps"], g["weight_decay"], self._step,
                                   max_norm if (max_norm is not None and max_norm > 0 and n_part != 0) else 0.0))
        if self._inv_scale is not None:           # device-side 1/scale (no host read of the GradScaler's scale)
            self._hp[K.HP_INVSCALE:K.HP_INVSCALE + 1].copy_(self._inv_scale.reshape(1))
            self._inv_scale = None
        if self._zero is not None:
            self._zero.step(self._hp, _check_inf, self._flag, self._skipped, self.stats)   # gradients are zeroed by the kernel
            self._grads_synced = False
            return loss
        K.adamw_step(fv.own(fv.flat), fv.own(fv.grad), self.exp_avg, self.exp_avg_sq, fv.own_shadow(), self._hp,
                     self._partials, n_part, self._flag if _check_inf else None, self.stats,
                     zero_grad=self.zero_grad_in_step and not fv.sharded, skipped=self._skipped)
        fv.gather_compute_weights()
        if self.zero_grad_in_step and fv.sharded:
            fv.grad.zero_()
        self._grads_synced = False
        return loss

    def zero_grad(self, set_to_none: bool = False) -> None:
        # gradients are views of the flat accumulator: keep them, zero in one op (reference: optimizer.zero_grad(),
        # train_fsdp.py:408).  With zero_grad_in_step the kernel already did it.
        if not self.zero_grad_in_step and self._zero is None:
            self.fv.grad.zero_()
        self._grads_synced = False


def clip_grad_norm_(target, max_norm: float, optimizer: FusedAdamW | None = None) -> torch.Tensor:
    """Global-norm clipping (reference: model.clip_grad_norm_(1.0) train_fsdp.py:395;
    torch.nn.utils.clip_grad_norm_ train_diloco_torch.py:323).

    With a FusedAdamW ``optimizer`` the scaling is deferred into the fused step (one norm pass, no extra sweep over
    the gradients); otherwise falls back to the torch utility on the given parameters."""
    if optimizer is not None and isinstance(optimizer, FusedAdamW):
        return optimizer.compute_grad_norm_partials(max_norm)
    if hasattr(target, "clip_grad_norm_"):
        return target.clip_grad_norm_(max_norm)
    params = target.parameters() if hasattr(target, "parameters") else target
    return torch.nn.utils.clip_grad_norm_(list(params), max_norm)
