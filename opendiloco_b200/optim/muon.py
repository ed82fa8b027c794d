"""``FusedMuon``: ``torch.optim.Muon`` on the hidden matrices and ``torch.optim.AdamW`` on everything else, over the flat
parameter buffer of ``FusedAdamW``.

Muon (Jordan et al. 2024; Liu et al. 2025, "Muon is Scalable for LLM Training") takes momentum, then orthogonalises each
weight matrix's update with a few Newton-Schulz iterations.  Here:

* Muon parameters are the ``q/k/v/o_proj`` and ``gate/up/down_proj`` weights of an arena-backed Llama, each its own
  matrix; on other modules every 2-D parameter.  Everything else (embedding, LM head, norm weights) gets AdamW.
* On CUDA, the matrices whose dimensions are multiples of 64 run the kernels of ``ops/muon.py``: one prepare launch
  (clip, momentum, per-chunk norm partials), then per shape group and bounded chunk a normalise/cast into a stacked
  bf16 scratch, ``ns_steps`` x 3 batched wgmma GEMMs, and one apply launch.  The AdamW parameters take one segmented
  launch.  Other matrices, and every parameter on CPU, run the PyTorch reference with the same rounding points.
* The Muon momentum lives in the flat ``exp_avg`` buffer on the matrix slots; the AdamW moments on the others.  Memory
  is FusedAdamW's plus the bounded Newton-Schulz scratch.
* Global-norm clipping, the ``model.clip_grad_norm_`` hand-off, GradScaler steps and NO_SHARD data parallelism work as
  in FusedAdamW, which this class extends.  ZeRO sharding is rejected: Muon needs whole matrices.
* Both groups' lr, the momentum, the weight decays, the AdamW betas / bias corrections, the clip threshold and the loss
  scale are read from device memory on every step (schedules need no re-capture).  ``ns_coefficients``, ``ns_steps``,
  ``eps`` and ``adjust_lr_fn`` are fixed at construction: they shape the launch sequence and the per-matrix tables.
"""
from __future__ import annotations

import math
import struct

import torch

from ..ops import kernels as K
from ..ops import muon as M
from .fused import FusedAdamW

MUON_NAMES = ("q_proj", "k_proj", "v_proj", "o_proj", "gate_proj", "up_proj", "down_proj")
CHUNK = 1 << 16                      # elements per prepare / AdamW chunk (one CTA each)
SCRATCH_BYTES = 512 << 20            # Newton-Schulz scratch: two X and two m x m bf16 buffers of SCRATCH_BYTES / 8 elements each
X_CAP = A_CAP = SCRATCH_BYTES // 8   # a shape group is processed in chunks that fit both capacities


def _is_muon_param(p: torch.nn.Parameter) -> bool:
    name = getattr(p, "_odb_name", None)
    if name is not None:
        return p.ndim == 2 and any(f".{k}." in name for k in MUON_NAMES)
    return p.ndim == 2


def adjust_lr_ratio(adjust_lr_fn: str | None, shape) -> float:
    """torch.optim.Muon's learning-rate adjustment factor for a [A, B] matrix."""
    A, B = shape[:2]
    if adjust_lr_fn is None or adjust_lr_fn == "original":
        return math.sqrt(max(1.0, A / B))
    if adjust_lr_fn == "match_rms_adamw":
        return 0.2 * math.sqrt(max(A, B))
    raise ValueError(f"unknown adjust_lr_fn {adjust_lr_fn!r}")


def _chunks(spans: list[tuple[int, int]]) -> list[tuple[int, int]]:
    return [(o + s, min(CHUNK, n - s)) for o, n in spans for s in range(0, n, CHUNK)]


class FusedMuon(FusedAdamW):
    CHECKPOINT_KIND = "muon"             # utils/ckpt.py tags the shards with it; FusedAdamW checkpoints carry no tag
    def __init__(self, params, lr: float = 1e-3, weight_decay: float = 0.1, momentum: float = 0.95, nesterov: bool = True,
                 ns_coefficients: tuple[float, float, float] = (3.4445, -4.775, 2.0315), eps: float = 1e-7, ns_steps: int = 5,
                 adjust_lr_fn: str | None = None, adamw_lr: float | None = None, adamw_betas=(0.9, 0.95), adamw_eps: float = 1e-8,
                 max_grad_norm: float | None = None, zero_grad_in_step: bool = False, dp_group=None, shard: bool = False,
                 shard_params: bool = False):
        if shard or shard_params:
            raise ValueError("FusedMuon needs whole matrices: ZeRO sharding (shard=True) is not supported")
        if adjust_lr_fn not in (None, "original", "match_rms_adamw"):
            raise ValueError(f"unknown adjust_lr_fn {adjust_lr_fn!r}")
        if not 0 <= ns_steps < 100 or len(ns_coefficients) != 3:
            raise ValueError("ns_steps must be in [0, 100) and ns_coefficients hold three values")
        params = list(params)
        if params and isinstance(params[0], dict):
            params = [p for g in params for p in g["params"]]
        adamw_lr = lr if adamw_lr is None else adamw_lr
        super().__init__(params, lr=adamw_lr, betas=adamw_betas, eps=adamw_eps, weight_decay=weight_decay,
                         max_grad_norm=max_grad_norm, zero_grad_in_step=zero_grad_in_step, dp_group=dp_group)
        fv = self.fv
        self._muon_idx = [i for i, p in enumerate(fv.params) if _is_muon_param(p)]
        self._adamw_idx = [i for i in range(len(fv.params)) if i not in set(self._muon_idx)]
        self.param_groups = [
            dict(params=[fv.params[i] for i in self._muon_idx], lr=lr, weight_decay=weight_decay, momentum=momentum,
                 nesterov=nesterov, ns_coefficients=tuple(ns_coefficients), eps=eps, ns_steps=ns_steps,
                 adjust_lr_fn=adjust_lr_fn),
            dict(params=[fv.params[i] for i in self._adamw_idx], lr=adamw_lr, betas=tuple(adamw_betas), eps=adamw_eps,
                 weight_decay=weight_decay),
        ]
        self.state.clear()
        self._init_state_views()
        self._ns = (tuple(float(c) for c in ns_coefficients), int(ns_steps), float(eps), adjust_lr_fn)   # construction-time
        self._ref_idx = self._muon_idx               # matrices on the reference path (narrowed by _make_plan on CUDA)
        self._plan = self._make_plan() if fv.flat.is_cuda else None
        self._scratch: list[torch.Tensor] | None = None

    # ----------------------------------------------------------------- kernel plan (CUDA)
    def _make_plan(self) -> dict:
        fv, dev = self.fv, self.fv.flat.device
        adjust_fn = self._ns[3]
        kern = [i for i in self._muon_idx if M.kernel_shape(*fv.params[i].shape)]
        self._ref_idx = [i for i in self._muon_idx if i not in set(kern)]
        prep_chunks, groups, mats, c = [], {}, [], 0
        for i in kern:
            p = fv.params[i]
            R, C = p.shape
            own = _chunks([(fv.offsets[i], p.numel())])
            prep_chunks += own
            adj = struct.unpack("<i", struct.pack("<f", adjust_lr_ratio(adjust_fn, p.shape)))[0] & 0xFFFFFFFF
            groups.setdefault((min(R, C), max(R, C)), []).append([fv.offsets[i], R, C, int(R > C), c, c + len(own), 0, adj])
            mats.append((c, c + len(own)))
            c += len(own)
        plan_groups, x_elems, a_elems = [], 0, 0
        for (m, n), rows in groups.items():
            per = max(1, min(X_CAP // (m * n), A_CAP // (m * m)))
            for s in range(0, len(rows), per):
                part = rows[s:s + per]
                for j, r in enumerate(part):
                    r[6] = j * m * n
                plan_groups.append((m, n, len(part), torch.tensor(part, dtype=torch.int64, device=dev)))
                x_elems, a_elems = max(x_elems, len(part) * m * n), max(a_elems, len(part) * m * m)
        aw = _chunks([(fv.offsets[i], fv.params[i].numel()) for i in self._adamw_idx])
        return dict(
            prep=torch.tensor(prep_chunks, dtype=torch.int64, device=dev).reshape(-1, 2) if prep_chunks else None,
            upart=torch.zeros(max(1, len(prep_chunks)), dtype=torch.float32, device=dev),
            mats=torch.tensor(mats, dtype=torch.int64, device=dev).reshape(-1, 2) if mats else None,
            scale=torch.zeros(2 * max(1, len(prep_chunks)), dtype=torch.float32, device=dev),
            groups=plan_groups, x_elems=x_elems, a_elems=a_elems,
            adamw=torch.tensor(aw, dtype=torch.int64, device=dev).reshape(-1, 2) if aw else None)

    def _ns_scratch(self) -> list[torch.Tensor]:
        if self._scratch is None:
            dev, pl = self.fv.flat.device, self._plan
            self._scratch = [torch.empty(pl[k], dtype=torch.bfloat16, device=dev) for k in ("x_elems", "x_elems", "a_elems", "a_elems")]
        return self._scratch

    # ----------------------------------------------------------------- torch-compatible per-param state
    def _init_state_views(self) -> None:
        if not hasattr(self, "_muon_idx"):          # FusedAdamW.__init__ runs before the groups are split
            return super()._init_state_views()
        fv = self.fv
        for i in self._muon_idx:
            self.state[fv.params[i]] = {"momentum_buffer": fv.view_of(self.exp_avg, i)}
        for i in self._adamw_idx:
            self.state[fv.params[i]] = {"step": torch.tensor(float(self._step)), "exp_avg": fv.view_of(self.exp_avg, i),
                                        "exp_avg_sq": fv.view_of(self.exp_avg_sq, i)}

    def state_dict(self):
        step = self.applied_steps()
        for st in self.state.values():
            if "step" in st:
                st["step"] = torch.tensor(float(step))
        return torch.optim.Optimizer.state_dict(self)

    def load_state_dict(self, state_dict) -> None:
        torch.optim.Optimizer.load_state_dict(self, state_dict)
        fv, step = self.fv, self.applied_steps()
        for i in self._muon_idx:
            st = self.state.get(fv.params[i], {})
            if "momentum_buffer" in st:
                fv.view_of(self.exp_avg, i).copy_(st["momentum_buffer"])
        for i in self._adamw_idx:
            st = self.state.get(fv.params[i], {})
            if "exp_avg" in st:
                fv.view_of(self.exp_avg, i).copy_(st["exp_avg"])
                fv.view_of(self.exp_avg_sq, i).copy_(st["exp_avg_sq"])
                step = int(float(st.get("step", 0)))
        self.restore_step_count(step)
        self.state.clear()
        self._init_state_views()

    # ----------------------------------------------------------------- step
    @torch.no_grad()
    def step(self, closure=None, _check_inf: bool = False):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        self.sync_grads()
        fv = self.fv
        mg, ag = self.param_groups
        self._step += 1
        max_norm = self.max_grad_norm
        n_part = 0
        if self._pending is not None:
            n_part, max_norm = self._pending
            self._pending = None
        elif (max_norm is not None and max_norm > 0) or _check_inf:
            n_part = self._norm_partials()
        hp = K.adamw_hp(ag["lr"], ag["betas"], ag["eps"], ag["weight_decay"], self._step,
                        max_norm if (max_norm is not None and max_norm > 0 and n_part != 0) else 0.0)
        hp.update({M.HP_MLR: mg["lr"], M.HP_MOM: mg["momentum"], M.HP_MWD: mg["weight_decay"],
                   M.HP_NESTEROV: float(bool(mg["nesterov"]))})
        self._upload_hp(hp)
        if self._inv_scale is not None:
            self._hp[K.HP_INVSCALE:K.HP_INVSCALE + 1].copy_(self._inv_scale.reshape(1))
            self._inv_scale = None
        flag = self._flag if _check_inf else None
        zero = self.zero_grad_in_step
        if self._plan is not None:
            self._step_cuda(mg, n_part, flag, zero)
        else:
            for i in self._adamw_idx:
                sl = slice(fv.offsets[i], fv.offsets[i] + fv.params[i].numel())
                K.adamw_step(fv.flat[sl], fv.grad[sl], self.exp_avg[sl], self.exp_avg_sq[sl],
                             None if fv.shadow is None else fv.shadow[sl], self._hp, self._partials, n_part, flag, self.stats,
                             zero_grad=zero, skipped=self._skipped)
        self._step_reference(mg, n_part, flag, zero)
        self._grads_synced = False
        return loss

    def _step_cuda(self, mg: dict, n_part: int, flag, zero: bool) -> None:
        fv, pl = self.fv, self._plan
        if pl["adamw"] is not None:
            M.adamw_segments(fv.flat, fv.grad, self.exp_avg, self.exp_avg_sq, fv.shadow, pl["adamw"], self._hp, self._partials,
                             n_part, flag, zero, skipped=self._skipped)
        if pl["prep"] is None:
            return
        coeffs, steps, eps, _ = self._ns
        M.muon_prepare(fv.grad, self.exp_avg, pl["prep"], self._hp, self._partials, n_part, flag, pl["upart"], self.stats)
        M.muon_scale(pl["mats"], self._hp, self._partials, n_part, pl["upart"], pl["scale"], eps)
        x_all, x2_all, a_all, b_all = self._ns_scratch()
        for m, n, k, table in pl["groups"]:
            x, x2 = x_all[:k * m * n].view(k, m, n), x2_all[:k * m * n].view(k, m, n)
            am, bm = a_all[:k * m * m].view(k, m, m), b_all[:k * m * m].view(k, m, m)
            M.muon_normalize(fv.grad, self.exp_avg, table, m, n, self._hp, pl["scale"], x)
            out = M.newton_schulz(x, coeffs, steps, x2, am, bm)
            M.muon_apply(fv.flat, fv.grad, fv.shadow, table, m, n, self._hp, out, flag, zero)

    def _step_reference(self, mg: dict, n_part: int, flag, zero: bool) -> None:
        """The Muon matrices the kernels do not cover (all of them on CPU), on their own device."""
        if not self._ref_idx:
            return
        fv = self.fv
        coef = M.clip_coef_ref(self._hp, self._partials, n_part, self.stats)
        skip = flag is not None and int(flag.item()) != 0
        for i in self._ref_idx:
            p = fv.params[i]
            sl = slice(fv.offsets[i], fv.offsets[i] + p.numel())
            M.muon_update_ref(fv.view_of(fv.flat, i), fv.view_of(fv.grad, i), fv.view_of(self.exp_avg, i),
                              None if fv.shadow is None else fv.shadow[sl].view(p.shape), coef, mg["lr"], mg["weight_decay"],
                              mg["momentum"], mg["nesterov"], self._ns[0], self._ns[1], self._ns[2],
                              adjust_lr_ratio(self._ns[3], p.shape), skip)
            if zero:
                fv.grad[sl].zero_()
