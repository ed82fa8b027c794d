"""Checkpoint / resume (reference: open_diloco/ckpt_utils.py; SURVEY.md §3.5, §5.4).

On-disk layout is the reference's:

    <ckpt.path>/model_step_<N>/[diloco_rank_<r>/]
        .metadata                 JSON: flat-arena layout + shard table          (reference: DCP metadata)
        __<rank>_0.distcp         this rank's shard of {"model","optimizer"} ...  (reference: DCP shards, ckpt_utils.py:77-82)
        __<rank>_0.pt             {"data_loader": loader.state_dict()}            (ckpt_utils.py:83-87)
        global_state_dict.pt      {"scheduler","loss","outer_optimizer"?,"scaler"?}  (ckpt_utils.py:93-100)

with two deliberate additions the reference lacks (SURVEY.md §5.4 "what is not saved"): the outer parameters
theta_outer (+ momentum) and the inner-step phase (samples accumulated towards the next outer step), so resuming at a
step that is not a multiple of ``local_steps`` does not silently move the outer anchor.

Shards are flat slices ``[lo, hi)`` of the parameter arena, so a checkpoint written with one sharding degree can be
read back with another (ranges are re-assembled on load).  All file access goes through fsspec (``gs://`` etc. work).
"""
from __future__ import annotations

import io
import json
import os

import fsspec
import torch
from fsspec.generic import GenericFileSystem

from .config import BaseConfig
from .logger import get_logger

GLOBAL_STATE_FILE = "global_state_dict.pt"
CKPT_PREFIX = "model_step"
METADATA_FILE = ".metadata"

logger = get_logger()


class CkptConfig(BaseConfig):
    resume: str | bool | None = None   # True => newest model_step_* under `path`; str => that checkpoint directory
    interval: int | None = None
    path: str = "outputs"
    topk: int | None = None


# ------------------------------------------------------------------------------------------------ discovery / GC
def filter_ckpt_files(f: str) -> bool:
    if CKPT_PREFIX not in f:
        return False
    try:
        int(f.split("_")[-1])
        return True
    except ValueError:
        return False


def _list_ckpts(path: str) -> list[str]:
    fs = GenericFileSystem()
    return [f for f in fs.ls(path, detail=False) if filter_ckpt_files(f.rstrip("/"))]


def get_resume_info(ckpt_config: CkptConfig) -> tuple[bool, str | None]:
    """(should_resume, checkpoint_dir).  ``resume=True`` picks the checkpoint with the largest step suffix."""
    if ckpt_config.resume is None or ckpt_config.resume is False:
        return False, None
    if isinstance(ckpt_config.resume, bool):
        try:
            files = _list_ckpts(ckpt_config.path)
        except FileNotFoundError:
            logger.info(f"Checkpoint path {ckpt_config.path} not found, starting from scratch")
            return False, None
        if not files:
            logger.info(f"No checkpoints found in {ckpt_config.path}, starting from scratch")
            return False, None
        return True, max(files, key=lambda f: int(f.rstrip("/").split("_")[-1]))
    return True, ckpt_config.resume


def delete_old_checkpoints(checkpoint_path: str, topk: int) -> list[str]:
    fs = GenericFileSystem()
    files = sorted(_list_ckpts(checkpoint_path), key=lambda x: int(x.rstrip("/").split("_")[-1]))
    deleted = []
    for f in files[:-topk] if topk > 0 else files:
        fs.rm(f, recursive=True)
        deleted.append(f)
    return deleted


def get_diloco_rank_dir_name(world_rank_diloco: int) -> str:
    return f"diloco_rank_{world_rank_diloco}"


def check_checkpoint_path_access(checkpoint_path: str, rank: int, world_rank_hv: int | None = None) -> None:
    """Fail fast if the checkpoint location is not writable (reference ckpt_utils.py:182-193; unlike the reference,
    worker 0 also probes its own diloco_rank_0 directory - SURVEY.md §2.7)."""
    base = checkpoint_path if world_rank_hv is None else os.path.join(checkpoint_path, get_diloco_rank_dir_name(world_rank_hv))
    dummy = os.path.join(base, f"dummy_file_{rank}.txt")
    with fsspec.open(dummy, "w", auto_mkdir=True) as f:
        f.write("This is a dummy file for testing access.")
    GenericFileSystem().rm(dummy)


# ------------------------------------------------------------------------------------------------ io helpers
def _save(obj, path: str) -> None:
    buf = io.BytesIO()
    torch.save(obj, buf)
    with fsspec.open(path, "wb", auto_mkdir=True) as f:
        f.write(buf.getvalue())


def _load(path: str):
    with fsspec.open(path, "rb") as f:
        return torch.load(io.BytesIO(f.read()), map_location="cpu", weights_only=False)


def _inner_of(optimizer):
    return getattr(optimizer, "inner_optimizer", optimizer)


def _flat_view(optimizer):
    return getattr(_inner_of(optimizer), "fv", None)


def inner_kind(optimizer) -> str:
    """``"muon"`` for FusedMuon, ``"adamw"`` otherwise.  Flat shards of both look alike (exp_avg holds Muon's momentum on
    the matrix slots), so Muon checkpoints carry the tag and a resume under the other optimizer is refused."""
    return getattr(_inner_of(optimizer), "CHECKPOINT_KIND", "adamw")


def check_inner_kind(saved: str, optimizer) -> None:
    ours = inner_kind(optimizer)
    if saved != ours:
        raise ValueError(f"checkpoint was written by the {saved!r} inner optimizer; it cannot be resumed with {ours!r}")


# ------------------------------------------------------------------------------------------------ save
def save_checkpoint(checkpoint_path: str, model: torch.nn.Module, optimizer: torch.optim.Optimizer, scheduler=None,
                    outer_optimizer: torch.optim.Optimizer | None = None, scaler=None, loss: float | None = None,
                    data_loader=None, save_global_state: bool = True, diloco=None, rank: int | None = None) -> None:
    """Write one checkpoint directory.  ``optimizer`` is the INNER optimizer (FusedAdamW or any torch optimizer),
    ``outer_optimizer`` the outer torch optimizer, ``diloco`` the DiLoCoOptimizer (for theta_outer and the phase).
    ``rank`` = rank inside the worker (defaults to $RANK like the reference)."""
    rank = int(os.environ.get("RANK", 0)) if rank is None else rank
    fv = _flat_view(optimizer)
    inner = _inner_of(optimizer)
    shard: dict = {"format": "opendiloco_b200.flat.v1"}
    kind = inner_kind(optimizer)
    if kind != "adamw":
        shard["inner_optimizer"] = kind
    if fv is not None:
        lo, hi = fv.lo, fv.hi
        writes = fv.sharded or rank == 0
        if writes:
            shard.update(lo=lo, hi=hi, numel=fv.numel, model=fv.flat[lo:hi].detach().cpu(),
                         exp_avg=inner.exp_avg.detach().cpu(), exp_avg_sq=inner.exp_avg_sq.detach().cpu(),
                         step=inner.applied_steps(), param_groups=[{k: v for k, v in g.items() if k != "params"} for g in inner.param_groups])
            if diloco is not None:
                sa = diloco.state_averager
                if hasattr(diloco, "_sync_outer_state"):
                    diloco._sync_outer_state()      # sharded fused outer step: wait for the background momentum all-gather
                shard["theta_outer"] = sa.theta_outer.detach().cpu()
                if sa.momentum_buffer is not None:
                    shard["outer_momentum"] = sa.momentum_buffer.detach().cpu()
            _save(shard, os.path.join(checkpoint_path, f"__{rank}_0.distcp"))
        if rank == 0:
            arena = getattr(model, "arena", None)
            meta = {"format": shard["format"], "numel": fv.numel, "sharded": bool(fv.sharded),
                    "slots": {n: [s.offset, list(s.shape)] for n, s in arena.slots.items()} if arena is not None else None}
            if kind != "adamw":
                meta["inner_optimizer"] = kind
            with fsspec.open(os.path.join(checkpoint_path, METADATA_FILE), "w", auto_mkdir=True) as f:
                json.dump(meta, f)
    elif rank == 0:   # generic torch model/optimizer
        shard.update(model_state_dict=model.state_dict(), optimizer_state_dict=inner.state_dict())
        _save(shard, os.path.join(checkpoint_path, f"__{rank}_0.distcp"))
    if data_loader is not None and hasattr(data_loader, "state_dict"):
        _save({"data_loader": data_loader.state_dict()}, os.path.join(checkpoint_path, f"__{rank}_0.pt"))
    if not save_global_state:
        return
    g: dict = {"scheduler": scheduler.state_dict() if scheduler is not None else None, "loss": loss if loss is not None else 0}
    if outer_optimizer is not None:
        sd = outer_optimizer.state_dict()
        g["outer_optimizer"] = {"param_groups": sd["param_groups"],
                                "state": {} if fv is not None else sd["state"]}   # flat tensors live in the shard files
    if diloco is not None:
        g["diloco"] = {"local_epoch": diloco.local_epoch, "samples_accumulated": diloco.tracker.local_progress.samples_accumulated,
                       "drifted": bool(getattr(diloco, "_drifted", False))}
    if scaler is not None:
        g["scaler"] = scaler.state_dict()
    _save(g, os.path.join(checkpoint_path, GLOBAL_STATE_FILE))


# ------------------------------------------------------------------------------------------------ load
_SHARD_CACHE: dict[str, dict] = {}      # shard files of the checkpoint being loaded (cleared by load_checkpoint)


def _load_shard(path: str) -> dict:
    sh = _SHARD_CACHE.get(path)
    if sh is None:
        sh = _SHARD_CACHE[path] = _load(path)
    return sh


def _assemble(checkpoint_path: str, key: str, lo: int, hi: int, device) -> torch.Tensor | None:
    """Collect flat range [lo, hi) of ``key`` from whichever shard files cover it (every file is read once per load)."""
    fs = GenericFileSystem()
    files = [f for f in fs.ls(checkpoint_path, detail=False) if f.endswith(".distcp")]
    out = torch.empty(hi - lo, dtype=torch.float32)
    covered = 0
    for f in sorted(files):
        sh = _load_shard(f)
        if key not in sh:
            continue
        slo, shi = sh["lo"], sh["hi"]
        a, b = max(lo, slo), min(hi, shi)
        if a < b:
            out[a - lo:b - lo].copy_(sh[key][a - slo:b - slo])
            covered += b - a
    if covered == 0:
        return None
    if covered != hi - lo:
        raise RuntimeError(f"checkpoint {checkpoint_path} covers only {covered} of {hi - lo} elements of {key}")
    return out.to(device)


def load_checkpoint(checkpoint_path: str, model: torch.nn.Module, optimizer: torch.optim.Optimizer, scheduler=None,
                    outer_optimizer: torch.optim.Optimizer | None = None, scaler=None, data_loader=None, diloco=None,
                    rank: int | None = None) -> float:
    """Restore everything ``save_checkpoint`` wrote; returns the stored loss (reference ckpt_utils.py:103-156)."""
    rank = int(os.environ.get("RANK", 0)) if rank is None else rank
    fv = _flat_view(optimizer)
    inner = _inner_of(optimizer)
    _SHARD_CACHE.clear()
    if fv is not None:
        first = _load_shard(sorted(f for f in GenericFileSystem().ls(checkpoint_path, detail=False) if f.endswith(".distcp"))[0])
        check_inner_kind(first.get("inner_optimizer", "adamw"), optimizer)
        dev = fv.flat.device
        fv.flat[fv.lo:fv.hi].copy_(_assemble(checkpoint_path, "model", fv.lo, fv.hi, dev))
        m, v = _assemble(checkpoint_path, "exp_avg", fv.lo, fv.hi, dev), _assemble(checkpoint_path, "exp_avg_sq", fv.lo, fv.hi, dev)
        if m is not None:
            inner.exp_avg.copy_(m)
            inner.exp_avg_sq.copy_(v)
        inner.restore_step_count(int(first.get("step", 0)))
        # publish the restored weights to the compute copy (and to the worker's other GPUs when sharded)
        arena = getattr(model, "arena", None)
        if fv.sharded:
            import torch.distributed as dist

            dist.all_gather_into_tensor(fv.flat, fv.flat[fv.lo:fv.hi].clone(), group=fv.shard_group)
        if arena is not None:
            arena.sync_shadow()
        if diloco is not None:
            sa = diloco.state_averager
            to = _assemble(checkpoint_path, "theta_outer", fv.lo, fv.hi, sa.theta_outer.device)
            sa.theta_outer.copy_(to if to is not None else sa.theta_local)
            mom = _assemble(checkpoint_path, "outer_momentum", fv.lo, fv.hi, sa.theta_outer.device)
            if mom is not None and sa.momentum_buffer is not None:
                sa.momentum_buffer.copy_(mom)
    else:
        sh = _load(os.path.join(checkpoint_path, "__0_0.distcp"))
        check_inner_kind(sh.get("inner_optimizer", "adamw"), optimizer)
        model.load_state_dict(sh["model_state_dict"])
        inner.load_state_dict(sh["optimizer_state_dict"])
    if data_loader is not None and hasattr(data_loader, "load_state_dict"):
        data_loader.load_state_dict(_load(os.path.join(checkpoint_path, f"__{rank}_0.pt"))["data_loader"])
    g = _load(os.path.join(checkpoint_path, GLOBAL_STATE_FILE))
    if scheduler is not None and g.get("scheduler") is not None:
        scheduler.load_state_dict(g["scheduler"])
        for grp, lr in zip(inner.param_groups, scheduler.get_last_lr()):  # reference ckpt_utils.py:149-151, every group
            grp["lr"] = lr
    if outer_optimizer is not None and "outer_optimizer" in g:
        for grp, saved in zip(outer_optimizer.param_groups, g["outer_optimizer"]["param_groups"]):
            grp.update({k: v for k, v in saved.items() if k != "params"})
        if fv is None and g["outer_optimizer"]["state"]:
            outer_optimizer.load_state_dict(g["outer_optimizer"])
    if diloco is not None and "diloco" in g:
        diloco.state_averager.local_epoch = int(g["diloco"]["local_epoch"])
        diloco._drifted = bool(g["diloco"].get("drifted", False))      # a resumed worker still asks for the drift repair
        diloco.tracker.update_epoch(diloco.local_epoch)
        diloco.tracker.report_local_progress(diloco.local_epoch, int(g["diloco"]["samples_accumulated"]))
    if scaler is not None and "scaler" in g:
        scaler.load_state_dict(g["scaler"])
    _SHARD_CACHE.clear()
    return g["loss"]
