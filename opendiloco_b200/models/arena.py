"""Flat parameter arena: every model tensor lives in ONE contiguous buffer per role.

  master  fp32 [P]   - the optimizer's weights (theta_local of DiLoCo)
  shadow  bf16 [P]   - compute weights read by the GEMMs (re-written by the fused AdamW / outer kernels)
  grad    fp32 [P]   - gradient accumulator (wgrad GEMMs accumulate straight into it)

There is no transposed copy of the weights: the dgrad GEMMs read ``shadow`` in its forward [out, in] layout as an MN-major
wgmma operand (``ops.tc_gemm.linear_nn``).

One buffer => one fused optimizer launch, one collective per outer step (the reference sends 111 per-tensor
messages: train_diloco_torch.py:342-346, SURVEY.md §2.5 N2), and q|k|v / gate|up weights that are physically
adjacent so a single GEMM covers them.  ``nn.Parameter`` objects handed to user code are *views* into ``master`` with
``.grad`` views into ``grad`` and carry the HF state-dict names (SURVEY.md Appendix B).
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

from ..ops import kernels as K
from .config import LlamaConfig

ALIGN = 128          # elements: every fusion group starts 512-B (fp32) / 256-B (bf16) aligned -> TMA / 16-B vectors
TOTAL_ALIGN = 16384  # elements: flat length is a multiple of this so 1/2/4/8-way shards stay vector aligned


@dataclass
class Slot:
    name: str
    shape: tuple
    offset: int
    numel: int


def llama_layout(cfg: LlamaConfig) -> list[list[tuple[str, tuple]]]:
    """Fusion groups in arena order; tensors inside a group are packed back-to-back."""
    h, i = cfg.hidden_size, cfg.intermediate_size
    groups: list[list[tuple[str, tuple]]] = [[("model.embed_tokens.weight", (cfg.vocab_size, h))]]
    for l in range(cfg.num_hidden_layers):
        p = f"model.layers.{l}."
        groups.append([(p + "input_layernorm.weight", (h,))])
        groups.append([
            (p + "self_attn.q_proj.weight", (cfg.q_dim, h)),
            (p + "self_attn.k_proj.weight", (cfg.kv_dim, h)),
            (p + "self_attn.v_proj.weight", (cfg.kv_dim, h)),
        ])
        groups.append([(p + "self_attn.o_proj.weight", (h, cfg.q_dim))])
        groups.append([(p + "post_attention_layernorm.weight", (h,))])
        groups.append([(p + "mlp.gate_proj.weight", (i, h)), (p + "mlp.up_proj.weight", (i, h))])
        groups.append([(p + "mlp.down_proj.weight", (h, i))])
    groups.append([("model.norm.weight", (h,))])
    groups.append([("lm_head.weight", (cfg.vocab_size, h))])
    return groups


def hf_param_order(cfg: LlamaConfig) -> list[str]:
    """Names in HF ``named_parameters()`` order (what torch optimizers / state dicts enumerate)."""
    names = ["model.embed_tokens.weight"]
    for l in range(cfg.num_hidden_layers):
        p = f"model.layers.{l}."
        names += [p + "self_attn.q_proj.weight", p + "self_attn.k_proj.weight", p + "self_attn.v_proj.weight",
                  p + "self_attn.o_proj.weight", p + "mlp.gate_proj.weight", p + "mlp.up_proj.weight",
                  p + "mlp.down_proj.weight", p + "input_layernorm.weight", p + "post_attention_layernorm.weight"]
    names += ["model.norm.weight", "lm_head.weight"]
    return names


class ParamArena:
    def __init__(self, cfg: LlamaConfig, device, compute_dtype: torch.dtype = torch.bfloat16):
        self.cfg = cfg
        self.compute_dtype = compute_dtype
        self.slots: dict[str, Slot] = {}
        off = 0
        for group in llama_layout(cfg):
            off = (off + ALIGN - 1) // ALIGN * ALIGN
            for name, shape in group:
                n = 1
                for s in shape:
                    n *= s
                self.slots[name] = Slot(name, tuple(shape), off, n)
                off += n
        self.used = off
        self.numel = (off + TOTAL_ALIGN - 1) // TOTAL_ALIGN * TOTAL_ALIGN
        self.version = 0             # bumped whenever master / grad / shadow move to another allocation (graph invalidation)
        # FULL_SHARD / HYBRID_SHARD (ZeRO-3): between uses only this rank's slice of the compute weights is kept
        self.param_group = None
        self.shadow_shard: torch.Tensor | None = None
        self.param_lo = self.param_hi = 0
        self._alloc(torch.device(device))

    # ------------------------------------------------------------------ storage
    def _alloc(self, device: torch.device) -> None:
        self.device = device
        self.master = torch.zeros(self.numel, dtype=torch.float32, device=device)
        self.grad = torch.zeros(self.numel, dtype=torch.float32, device=device)
        if self.compute_dtype == torch.float32:
            self.shadow = self.master
        else:
            self.shadow = torch.zeros(self.numel, dtype=self.compute_dtype, device=device)

    def migrate(self, device: torch.device) -> None:
        assert self.param_group is None, "move the model before the optimizer shards its parameters"
        old_master, old_grad = self.master, self.grad
        self._alloc(device)
        self.master.copy_(old_master)
        self.grad.copy_(old_grad)
        self.sync_shadow()

    def adopt_master(self, buf: torch.Tensor) -> None:
        """Re-home the master weights into an externally allocated buffer (e.g. an NVLink symmetric-memory window)."""
        assert buf.numel() == self.numel and buf.dtype == torch.float32
        buf.copy_(self.master)
        if self.shadow is self.master:
            self.shadow = buf
        self.master = buf
        self.version += 1

    # ------------------------------------------------------------------ parameter sharding (FULL_SHARD / HYBRID_SHARD)
    def enable_param_sharding(self, group, lo: int, hi: int) -> None:
        """ZeRO-3 for the compute weights, with the reference's granularity: FSDP wraps the whole model in ONE unit
        (train_fsdp.py:239-245, no auto-wrap policy), so the unit of gathering is the whole flat parameter - all-gathered
        before forward, freed ("resharded") after it, all-gathered again before backward, freed after it.  Between uses a
        rank holds only ``shadow_shard`` = its [lo, hi) slice (what the fused AdamW / outer kernels write)."""
        if self.shadow is self.master:
            return                                   # fp32 compute: the master weights are the compute weights
        self.param_group, self.param_lo, self.param_hi = group, lo, hi
        self.shadow_shard = self.shadow[lo:hi].clone()
        self.shadow = None

    @property
    def param_sharded(self) -> bool:
        return self.param_group is not None

    def materialize_shadow(self) -> None:
        """All-gather the full compute weights from the ranks' shards (no-op unless parameters are sharded)."""
        if self.param_group is None or self.shadow is not None:
            return
        import torch.distributed as dist

        full = torch.empty(self.numel, dtype=self.compute_dtype, device=self.device)
        dist.all_gather_into_tensor(full, self.shadow_shard, group=self.param_group)
        self.shadow = full

    def release_shadow(self) -> None:
        """Reshard: drop the gathered copy (the caching allocator gets the block back)."""
        if self.param_group is not None:
            self.shadow = None

    def sync_shadow(self) -> None:
        if self.param_group is not None:
            src = self.master[self.param_lo:self.param_hi]
            K.cast_to_bf16(src, self.shadow_shard) if self.shadow_shard.dtype == torch.bfloat16 else self.shadow_shard.copy_(src)
            self.shadow = None
            return
        if self.shadow is not self.master:
            if self.shadow.dtype == torch.bfloat16:
                K.cast_to_bf16(self.master, self.shadow)
            else:
                self.shadow.copy_(self.master)

    # ------------------------------------------------------------------ views
    def _view(self, buf: torch.Tensor, name: str) -> torch.Tensor:
        s = self.slots[name]
        return buf[s.offset:s.offset + s.numel].view(s.shape)

    def p(self, name: str) -> torch.Tensor:
        return self._view(self.master, name)

    def w(self, name: str) -> torch.Tensor:
        return self._view(self._full_shadow(), name)

    def _full_shadow(self) -> torch.Tensor:
        if self.shadow is None:
            raise RuntimeError("compute weights are sharded (FULL_SHARD): call arena.materialize_shadow() around their use")
        return self.shadow

    def g(self, name: str) -> torch.Tensor:
        return self._view(self.grad, name)

    def _fused(self, buf: torch.Tensor, first: str, rows: int, cols: int) -> torch.Tensor:
        s = self.slots[first]
        return buf[s.offset:s.offset + rows * cols].view(rows, cols)

    def qkv_w(self, l: int) -> torch.Tensor:
        return self._fused(self._full_shadow(), f"model.layers.{l}.self_attn.q_proj.weight", self.cfg.qkv_dim, self.cfg.hidden_size)

    def qkv_g(self, l: int) -> torch.Tensor:
        return self._fused(self.grad, f"model.layers.{l}.self_attn.q_proj.weight", self.cfg.qkv_dim, self.cfg.hidden_size)

    def gu_w(self, l: int) -> torch.Tensor:
        return self._fused(self._full_shadow(), f"model.layers.{l}.mlp.gate_proj.weight", 2 * self.cfg.intermediate_size,
                           self.cfg.hidden_size)

    def gu_g(self, l: int) -> torch.Tensor:
        return self._fused(self.grad, f"model.layers.{l}.mlp.gate_proj.weight", 2 * self.cfg.intermediate_size,
                           self.cfg.hidden_size)

    # ------------------------------------------------------------------ init (HF LlamaPreTrainedModel._init_weights)
    @torch.no_grad()
    def init_weights(self, seed: int | None = None) -> None:
        gen = None
        if seed is not None:
            gen = torch.Generator(device="cpu").manual_seed(seed)
        self.master.zero_()
        for name in hf_param_order(self.cfg):
            v = self.p(name)
            if v.dim() == 1:
                v.fill_(1.0)
            else:
                cpu = torch.empty(v.shape, dtype=torch.float32).normal_(0.0, self.cfg.initializer_range, generator=gen)
                v.copy_(cpu)
        self.sync_shadow()
