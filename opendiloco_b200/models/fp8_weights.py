"""FP8 weight-only generation and scoring (``generate(fp8_weights=True)``, ``score(fp8_weights=True)``).

The q|k|v, o, gate|up and down projections of every decoder layer are quantised per output row to e4m3 (the rule of
:mod:`opendiloco_b200.ops.fp8w`), at the start of every call that asks for it: training updates the compute weights in
place, so a copy taken earlier could be stale.  The embedding, the RMSNorm weights and the LM head stay as they are.

Two copies are kept, at fixed addresses (captured decode graphs stay valid across calls):

  q, inv   e4m3 weights [L, N, K] and fp32 row factors [L, N]: read by the skinny-M GEMM of the decode steps (M <= 64)
  Ŵ        the dequantised weights q * inv in the compute dtype: read by the bf16 GEMMs wherever M > 64 (prefill, scoring,
           wide verify passes and beam steps), and by the whole program on CPU and non-bf16 models

so the quantised model is exactly the bf16 model with every projection weight replaced by Ŵ, and that program is the
oracle of every path.  Together they take 1.5x the bf16 bytes of the projections (about 2.9 GB at the 1b preset) while
the option is in use; training state (master, shadow, gradients, optimizer state, workspaces, graphs) is never touched.
"""
from __future__ import annotations

import torch

from ..ops import fp8w as FW
from ..ops import tc_gemm as TC
from ..ops.fp8 import E4M3

KINDS = ("qkv", "o", "gu", "down")


def arena_weight(ar, kind: str, l: int) -> torch.Tensor:
    """The compute weight [N, K] of projection ``kind`` of layer l."""
    if kind == "qkv":
        return ar.qkv_w(l)
    if kind == "gu":
        return ar.gu_w(l)
    name = {"o": "self_attn.o_proj.weight", "down": "mlp.down_proj.weight"}[kind]
    return ar.w(f"model.layers.{l}.{name}")


def _key(ar) -> tuple:
    return (ar.version, ar.shadow.data_ptr(), str(ar.device), ar.compute_dtype)


class FP8Weights:
    """q, inv and Ŵ of every projection, the quantiser's segment table and the skinny GEMM's split-K workspace."""

    def __init__(self, cfg, ar):
        L, dev, dt = cfg.num_hidden_layers, ar.device, ar.compute_dtype
        self.key = _key(ar)
        self.q, self.inv, self.deq, self.splits, self.skinny_ok = {}, {}, {}, {}, {}
        self.kernels = all(FW.quantize_rows_usable(arena_weight(ar, k, l)) for k in KINDS for l in range(L))
        sms = torch.cuda.get_device_properties(dev).multi_processor_count if dev.type == "cuda" else 1
        ws = tiles = 0
        for kind in KINDS:
            N, Kd = arena_weight(ar, kind, 0).shape
            self.q[kind] = torch.empty(L, N, Kd, dtype=E4M3, device=dev)
            self.inv[kind] = torch.empty(L, N, dtype=torch.float32, device=dev)
            self.deq[kind] = torch.empty(L, N, Kd, dtype=dt, device=dev)
            self.skinny_ok[kind] = self.kernels and FW.gemm_shape_ok(N, Kd, swiglu=kind == "gu")
            self.splits[kind] = FW.default_splits(N, Kd, sms) if self.skinny_ok[kind] else 1
            ws = max(ws, FW.workspace_floats(N, self.splits[kind]))
            tiles = max(tiles, N // FW.TILE_N)
        self.ws = torch.zeros(max(ws, 1), dtype=torch.float32, device=dev)
        self.counters = torch.zeros(max(tiles, 1), dtype=torch.int32, device=dev)
        self.segs = None
        if self.kernels:
            rows = []
            for kind in KINDS:
                for l in range(L):
                    w = arena_weight(ar, kind, l)
                    rows.append([w.data_ptr(), self.q[kind][l].data_ptr(), self.inv[kind][l].data_ptr(), self.deq[kind][l].data_ptr(),
                                 w.shape[0], w.shape[1]])
            self.segs = torch.tensor(rows, dtype=torch.int64).to(dev)
            self.max_rows = max(r[4] for r in rows)

    @property
    def token(self) -> int:
        """Identifies these buffers in the keys of captured graphs."""
        return self.q["qkv"].data_ptr()

    @torch.no_grad()
    def refresh(self, ar) -> None:
        """Quantise the current compute weights: one kernel launch on CUDA bf16 models, the reference otherwise."""
        if self.kernels:
            FW.quantize_rows(self.segs, self.segs.shape[0], self.max_rows, self.ws)
            return
        for kind in KINDS:
            for l in range(self.q[kind].shape[0]):
                q, inv = FW.quantize_rows_ref(arena_weight(ar, kind, l))
                self.q[kind][l].copy_(q)
                self.inv[kind][l].copy_(inv)
                self.deq[kind][l].copy_(FW.dequantize_rows(q, inv, self.deq[kind].dtype))

    def weight(self, kind: str, l: int) -> torch.Tensor:
        return self.deq[kind][l]

    def skinny(self, kind: str, x: torch.Tensor) -> bool:
        """Whether ``x @ W^T`` runs on the skinny FP8 GEMM (M <= 64 and shapes the kernel covers)."""
        return self.skinny_ok[kind] and x.shape[0] <= FW.MAX_M and TC.usable(x)

    def linear(self, kind: str, l: int, x: torch.Tensor, out: torch.Tensor, act: torch.Tensor | None = None) -> None:
        FW.linear(x, self.q[kind][l], self.inv[kind][l], out, self.splits[kind], self.ws, self.counters, act=act)


def fp8_weights(model) -> FP8Weights:
    """The model's FP8 weights, allocated on first use (again after the arena moves) and re-quantised on every call."""
    eng, ar = model.engine, model.arena
    st = eng.fp8_weights
    if st is None or st.key != _key(ar):
        eng.fp8_weights = None                        # free the old buffers before allocating the new ones
        st = eng.fp8_weights = FP8Weights(model.config, ar)
    st.refresh(ar)
    return st


def check_flag(fp8_weights) -> bool:
    if not isinstance(fp8_weights, bool):
        raise ValueError(f"fp8_weights must be True or False, got {fp8_weights!r}")
    return fp8_weights
