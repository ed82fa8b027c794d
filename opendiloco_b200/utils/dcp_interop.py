"""Checkpoint interchange with the reference's on-disk format.

The reference writes ``torch.distributed.checkpoint`` (DCP) directories: ``dcp.save({"model": ..., "optimizer": ...})`` of the
FSDP-wrapped HF model plus ``global_state_dict.pt`` (ckpt_utils.py:48-100).  This framework stores flat ``[lo, hi)`` slices of
the parameter arena per rank (``utils/ckpt.py``: one read per rank, re-shardable, carries theta_outer and the outer momentum).
The two functions below translate between them on one process, so a run can be moved in either direction:

    python scripts/convert_ckpt.py to-dcp   outputs/model_step_1000/diloco_rank_0  /tmp/ref_format
    python scripts/convert_ckpt.py from-dcp /tmp/ref_format  outputs/imported --model 150m

DCP layout written / read here: ``model`` = {HF parameter name: tensor}; ``optimizer`` = {"state": {HF name: {"exp_avg",
"exp_avg_sq", "step"}}, "param_groups": [{..., "params": [HF names]}]} - the fully-qualified-name form
``torch.distributed.checkpoint.state_dict.get_state_dict`` produces for an FSDP(use_orig_params) model.
"""
from __future__ import annotations

import glob
import json
import os
import shutil

import torch

from .ckpt import GLOBAL_STATE_FILE, METADATA_FILE, _load, _save


_LAYER_ORDER = ["self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight", "self_attn.o_proj.weight",
                "mlp.gate_proj.weight", "mlp.up_proj.weight", "mlp.down_proj.weight", "input_layernorm.weight",
                "post_attention_layernorm.weight"]


def hf_order(names) -> list[str]:
    """Arena slot names -> HF ``named_parameters()`` order (what torch optimizers index their state by)."""
    def key(n: str):
        if n == "model.embed_tokens.weight":
            return (0, 0, 0)
        if n.startswith("model.layers."):
            _, _, idx, rest = n.split(".", 3)
            return (1, int(idx), _LAYER_ORDER.index(rest))
        return (2, 0, 0 if n == "model.norm.weight" else 1)

    return sorted(names, key=key)


def _gather_flat(ckpt_dir: str) -> tuple[dict, dict[str, torch.Tensor]]:
    """Assemble the full flat vectors of a flat-shard checkpoint directory -> (metadata, {key: flat fp32 tensor})."""
    with open(os.path.join(ckpt_dir, METADATA_FILE)) as f:
        meta = json.load(f)
    if meta.get("inner_optimizer", "adamw") != "adamw":
        # the reference's layout holds AdamW moments only: Muon's momentum would be read back as exp_avg
        raise ValueError(f"{ckpt_dir} was written by the {meta['inner_optimizer']!r} inner optimizer; only AdamW checkpoints convert")
    n = int(meta["numel"])
    flat: dict[str, torch.Tensor] = {}
    step, groups = 0, None
    for path in sorted(glob.glob(os.path.join(ckpt_dir, "__*_0.distcp"))):
        sh = _load(path)
        lo, hi = int(sh["lo"]), int(sh["hi"])
        step, groups = int(sh.get("step", step)), sh.get("param_groups", groups)
        for key in ("model", "exp_avg", "exp_avg_sq", "theta_outer", "outer_momentum"):
            if key in sh:
                flat.setdefault(key, torch.zeros(n, dtype=torch.float32))[lo:hi] = sh[key].to(torch.float32)
    meta["step"], meta["param_groups"] = step, groups
    return meta, flat


def export_dcp(ckpt_dir: str, out_dir: str) -> None:
    """Flat-shard checkpoint (one rank directory of ours) -> a DCP directory the reference's ``load_checkpoint`` reads."""
    import torch.distributed.checkpoint as dcp

    meta, flat = _gather_flat(ckpt_dir)
    slots = meta["slots"]
    if slots is None:
        raise ValueError("checkpoint was written for a non-arena model: nothing to name the tensors by")
    names = hf_order(slots)
    view = lambda buf, name: buf[slots[name][0]:slots[name][0] + int(torch.tensor(slots[name][1]).prod())].view(slots[name][1]).clone()  # noqa: E731
    model_sd = {name: view(flat["model"], name) for name in names}
    opt_state = {}
    if "exp_avg" in flat:
        for name in names:
            opt_state[name] = {"exp_avg": view(flat["exp_avg"], name), "exp_avg_sq": view(flat["exp_avg_sq"], name),
                               "step": torch.tensor(float(meta["step"]))}
    groups = [dict(g, params=names) for g in (meta["param_groups"] or [{}])]
    os.makedirs(out_dir, exist_ok=True)
    dcp.save({"model": model_sd, "optimizer": {"state": opt_state, "param_groups": groups}}, checkpoint_id=out_dir, no_dist=True)
    gpath = os.path.join(ckpt_dir, GLOBAL_STATE_FILE)
    if not os.path.isfile(gpath):                       # DiLoCo layout: the global file sits next to the rank directories
        gpath = os.path.join(os.path.dirname(ckpt_dir.rstrip("/")), GLOBAL_STATE_FILE)
    if os.path.isfile(gpath):
        g = _load(gpath)
        if "outer_optimizer" in g and "outer_momentum" in flat and not g["outer_optimizer"].get("state"):
            # torch SGD state is keyed by parameter index in named_parameters() order
            g["outer_optimizer"] = dict(g["outer_optimizer"],
                                        state={i: {"momentum_buffer": view(flat["outer_momentum"], name)} for i, name in enumerate(names)})
            g["outer_optimizer"]["param_groups"] = [dict(pg, params=list(range(len(names)))) for pg in g["outer_optimizer"]["param_groups"]]
        g.pop("diloco", None)                           # phase / theta_outer have no slot in the reference format
        _save(g, os.path.join(out_dir, GLOBAL_STATE_FILE))
    for extra in glob.glob(os.path.join(ckpt_dir, "__*_0.pt")):          # data-loader state, same file name in both formats
        shutil.copy(extra, out_dir)


def import_dcp(dcp_dir: str, out_dir: str, config) -> None:
    """A reference DCP checkpoint of a Llama with ``config`` -> a single-rank flat-shard directory ``load_checkpoint`` reads."""
    import torch.distributed.checkpoint as dcp

    from ..models.arena import ParamArena, hf_param_order

    arena = ParamArena(config, "cpu", torch.float32)
    names = hf_param_order(config)
    mk = lambda: {n: torch.zeros(arena.slots[n].shape) for n in names}  # noqa: E731
    template = {"model": mk(), "optimizer": {"state": {n: {"exp_avg": torch.zeros(arena.slots[n].shape),
                                                           "exp_avg_sq": torch.zeros(arena.slots[n].shape),
                                                           "step": torch.tensor(0.0)} for n in names},
                                             "param_groups": [{"lr": 0.0, "betas": (0.9, 0.95), "eps": 1e-8, "weight_decay": 0.1,
                                                               "params": list(names)}]}}
    dcp.load(template, checkpoint_id=dcp_dir, no_dist=True)
    flat = {k: torch.zeros(arena.numel) for k in ("model", "exp_avg", "exp_avg_sq")}
    for n in names:
        s = arena.slots[n]
        flat["model"][s.offset:s.offset + s.numel] = template["model"][n].reshape(-1).float()
        flat["exp_avg"][s.offset:s.offset + s.numel] = template["optimizer"]["state"][n]["exp_avg"].reshape(-1).float()
        flat["exp_avg_sq"][s.offset:s.offset + s.numel] = template["optimizer"]["state"][n]["exp_avg_sq"].reshape(-1).float()
    step = int(float(template["optimizer"]["state"][names[0]]["step"]))
    groups = [{k: v for k, v in g.items() if k != "params"} for g in template["optimizer"]["param_groups"]]
    os.makedirs(out_dir, exist_ok=True)
    _save({"format": "opendiloco_b200.flat.v1", "lo": 0, "hi": arena.numel, "numel": arena.numel, "step": step,
           "param_groups": groups, **flat}, os.path.join(out_dir, "__0_0.distcp"))
    with open(os.path.join(out_dir, METADATA_FILE), "w") as f:
        json.dump({"format": "opendiloco_b200.flat.v1", "numel": arena.numel, "sharded": False,
                   "slots": {n: [s.offset, list(s.shape)] for n, s in arena.slots.items()}}, f)
    gpath = os.path.join(dcp_dir, GLOBAL_STATE_FILE)
    if os.path.isfile(gpath):
        g = _load(gpath)
        if "outer_optimizer" in g and g["outer_optimizer"].get("state"):
            mom = torch.zeros(arena.numel)
            for i, n in enumerate(names):
                st = g["outer_optimizer"]["state"].get(i)
                if st is not None and st.get("momentum_buffer") is not None:
                    s = arena.slots[n]
                    mom[s.offset:s.offset + s.numel] = st["momentum_buffer"].reshape(-1).float()
            sh = _load(os.path.join(out_dir, "__0_0.distcp"))
            sh["outer_momentum"] = mom
            _save(sh, os.path.join(out_dir, "__0_0.distcp"))
            g["outer_optimizer"] = dict(g["outer_optimizer"], state={})
        _save(g, os.path.join(out_dir, GLOBAL_STATE_FILE))
    for extra in glob.glob(os.path.join(dcp_dir, "__*_0.pt")):
        shutil.copy(extra, out_dir)
