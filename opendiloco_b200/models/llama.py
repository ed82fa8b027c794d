"""Llama causal LM on the flat arena: hand-scheduled forward/backward over sm_90a kernels.

There is no autograd graph on the hot path.  ``LlamaEngine`` runs the layer program explicitly
(K1..K8 of SURVEY.md §2.5), keeps activations in shape-keyed static workspaces (CUDA-graph friendly) and
accumulates weight gradients straight into the fp32 gradient arena.  ``LlamaForCausalLM`` is the user-facing
``nn.Module``: HF-compatible parameter names / state dict / ``forward(input_ids, labels) -> .loss`` whose
``.backward()`` triggers the engine's backward through a single autograd node, so reference-style training loops
(train_fsdp.py:378-383, train_diloco_torch.py:312-318) run unchanged.

Op semantics follow the installed HF implementation the reference delegates to (SURVEY.md E1):
RMSNorm modeling_llama.py:62-67, RoPE :117-168, attention :251-289, MLP :182-184, decoder layer :303-332,
LM head + shifted CE :484-491 / loss_utils.py:45-67.
"""
from __future__ import annotations

import os
from dataclasses import dataclass
from pathlib import Path
from typing import Any

import torch
from torch import nn

from .. import _lib
from ..ops import attention as A
from ..ops import fp8 as F
from ..ops import gemm as G
from ..ops import kernels as K
from ..ops import tc_gemm as TC
from .arena import ParamArena, hf_param_order
from .config import LlamaConfig

IGNORE_INDEX = -100


def _use_graph() -> bool:
    """CUDA-graph replay of the micro-step (default on; ODB_CUDA_GRAPH=0 for the eager launch sequence): the thousands of
    short inter-kernel gaps of an eagerly launched step collapse into one graph launch (profiles/idle_gap.py measures it)."""
    return os.environ.get("ODB_CUDA_GRAPH", "1") == "1"



@dataclass
class CausalLMOutput:
    loss: torch.Tensor | None = None
    logits: torch.Tensor | None = None

    def __getitem__(self, k):
        return getattr(self, k) if isinstance(k, str) else (self.loss, self.logits)[k]


# ======================================================================================================= engine
class _Workspace:
    """Static activation buffers for one (B, S) shape."""

    def __init__(self, cfg: LlamaConfig, B: int, S: int, device, dtype, lce_chunk: int):
        T, h, i, L = B * S, cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers
        e = lambda *shape, dt=dtype: torch.empty(*shape, dtype=dt, device=device)  # noqa: E731
        f32 = torch.float32
        self.B, self.S, self.T = B, S, T
        self.ids = torch.empty(T, dtype=torch.int64, device=device)
        self.labels = torch.empty(T, dtype=torch.int64, device=device)      # HF-shifted labels
        self.labels_in = torch.empty(T, dtype=torch.int64, device=device)   # staging for host / strided label tensors
        # saved per layer
        self.xa = [e(T, h) for _ in range(L)]         # residual stream entering the attention block
        self.rstd1 = [e(T, dt=f32) for _ in range(L)]
        self.xn1 = [e(T, h) for _ in range(L)]
        self.qkv = [e(T, cfg.qkv_dim) for _ in range(L)]
        self.att = [None] * L                          # attention output (+aux) allocated by the attention op
        self.aux = [None] * L
        self.xm = [e(T, h) for _ in range(L)]         # residual stream entering the MLP block
        self.rstd2 = [e(T, dt=f32) for _ in range(L)]
        self.xn2 = [e(T, h) for _ in range(L)]
        self.gu = [e(T, 2 * i) for _ in range(L)]
        self.act = [e(T, i) for _ in range(L)]
        self.xf = e(T, h)                              # residual stream entering the final norm
        self.rstdf = e(T, dt=f32)
        self.xnf = e(T, h)
        # transient
        self.proj = e(T, h)                            # o-proj / down-proj output (the residual delta)
        self.dx = e(T, h)                              # gradient of the residual stream
        self.dn = e(T, h)                              # gradient w.r.t. a normed activation
        self.datt = e(T, h)
        self.dqkv = e(T, cfg.qkv_dim)
        self.dact = e(T, i)
        self.dxnf = e(T, h)
        self.lce_rows = min(lce_chunk, T)
        self._dev, self._dt, self._V = device, dtype, cfg.vocab_size
        self._logits = None          # reference path only (CPU / fp32 / fp16): bf16 kernels never materialise logits
        self._lce = None             # fused LCE buffers, allocated on first use
        self.loss_sum = torch.zeros(1, dtype=f32, device=device)
        self.gscale = torch.ones(1, dtype=f32, device=device)
        self.n_valid = torch.ones(1, dtype=f32, device=device)
        self.sumsq = torch.zeros(1, dtype=f32, device=device)
        self.cos, self.sin = K.rope_tables(S, cfg.head_dim, cfg.rope_theta, device)
        self.fp8: _Fp8Workspace | None = None      # precision="fp8-mixed" only

    @property
    def logits(self) -> torch.Tensor:
        if self._logits is None:
            self._logits = torch.empty(self.lce_rows, self._V, dtype=self._dt, device=self._dev)
        return self._logits

    def lce_buffers(self, planes: int, h: int):
        """(shift [T], rowscale [T], partials [2*planes, C], e [C, V] bf16, xs [C, h] bf16) of the fused LCE."""
        if self._lce is None:
            C, f32 = self.lce_rows, torch.float32
            mk = lambda *shape, dt: torch.empty(*shape, dtype=dt, device=self._dev)  # noqa: E731
            self._lce = (mk(self.T, dt=f32), mk(self.T, dt=f32), mk(2 * planes * C, dt=f32), mk(C, self._V, dt=self._dt),
                         mk(C, h, dt=self._dt))
        return self._lce


class _Fp8Workspace:
    """FP8 buffers of one (B, S) workspace (``precision="fp8-mixed"``, see ops/fp8.py for the recipe).

    Saved per layer: the transposed e4m3 copies of the four projection inputs (xn1, att, xn2, act), the K-major B operands
    of the weight gradients.  Transient: one row-major e4m3 activation copy, one row-major and one transposed e4m3 weight
    copy, and the row-major and transposed e5m2 copies of one gradient; each is consumed by the GEMMs right after its cast.
    Device scalars per layer (amax / inv, index = ``_F8_*``): four activations, four weights (the backward's transposed
    weight cast reuses the forward's amax), four gradients."""

    def __init__(self, cfg: LlamaConfig, T: int, device):
        h, I, L, qd, n_qkv = cfg.hidden_size, cfg.intermediate_size, cfg.num_hidden_layers, cfg.q_dim, cfg.qkv_dim
        e = lambda *shape, dt=F.E4M3: torch.empty(*shape, dtype=dt, device=device)  # noqa: E731
        self.T = T
        self.xn1_t = [e(h, T) for _ in range(L)]
        self.att_t = [e(qd, T) for _ in range(L)]
        self.xn2_t = [e(h, T) for _ in range(L)]
        self.act_t = [e(I, T) for _ in range(L)]
        self.a_row = e(T * max(h, qd, I))
        w_max = max(n_qkv * h, h * qd, 2 * I * h)
        self.w_row, self.w_t = e(w_max), e(w_max)
        g_max = T * max(h, 2 * I, n_qkv)
        self.g_row, self.g_t = e(g_max, dt=F.E5M2), e(g_max, dt=F.E5M2)
        self.amax = torch.zeros(L, 12, dtype=torch.float32, device=device)
        self.inv = torch.ones(L, 12, dtype=torch.float32, device=device)

    def _slot(self, l: int, i: int):
        return self.amax[l, i:i + 1], self.inv[l, i:i + 1]

    def act(self, l: int, i: int, x: torch.Tensor, x_t: torch.Tensor):
        """e4m3 copies of a projection input: row-major (transient, returned) and transposed (``x_t``, saved)."""
        T, n = x.shape
        row = self.a_row[: T * n].view(T, n)
        slot, inv = self._slot(l, i)
        F.quantize(x, slot, inv, F.E4M3, out=row, out_t=x_t)
        return row, inv

    def weight(self, l: int, i: int, w: torch.Tensor):
        """Row-major e4m3 copy of a compute weight for the forward GEMM."""
        row = self.w_row[: w.numel()].view(w.shape)
        slot, inv = self._slot(l, 4 + i)
        F.quantize(w, slot, inv, F.E4M3, out=row)
        return row, inv

    def weight_t(self, l: int, i: int, w: torch.Tensor):
        """Transposed e4m3 copy of a compute weight for the dgrad GEMM, scaled with the forward's amax."""
        t = self.w_t[: w.numel()].view(w.shape[1], w.shape[0])
        slot, inv = self._slot(l, 4 + i)
        F.cast(w, slot, F.E4M3, inv, out_t=t)
        return t, inv

    def grad(self, l: int, i: int, g: torch.Tensor):
        """e5m2 copies of a gradient: row-major (dgrad A operand) and transposed (weight-gradient A operand)."""
        T, n = g.shape
        row, t = self.g_row[: T * n].view(T, n), self.g_t[: T * n].view(n, T)
        slot, inv = self._slot(l, 8 + i)
        F.quantize(g, slot, inv, F.E5M2, out=row, out_t=t)
        return row, t, inv

    def act_inv(self, l: int, i: int) -> torch.Tensor:
        return self.inv[l, i:i + 1]


# slot indices of the four projection groups (activation i, weight 4 + i, gradient 8 + i)
_F8_QKV, _F8_O, _F8_GU, _F8_DOWN = 0, 1, 2, 3


class LlamaEngine:
    def __init__(self, cfg: LlamaConfig, arena: ParamArena, lce_chunk: int = 32768, fp8: bool = False):
        self.cfg, self.arena = cfg, arena
        # precision="fp8-mixed": the q|k|v, o, gate|up and down projections run as FP8 GEMMs (forward, dgrad, wgrad)
        self.fp8 = fp8
        # rows of the logits tile of the chunked linear-cross-entropy (ODB_LCE_CHUNK overrides: larger = fewer, fuller GEMM
        # launches and less reduce-add traffic into the lm_head gradient, at 64 KB of bf16 logits per row)
        self.lce_chunk = int(os.environ.get("ODB_LCE_CHUNK", lce_chunk))
        self._ws: dict[tuple, _Workspace] = {}
        self.collect_act_norms = False
        self.act_norms: dict[str, torch.Tensor] = {}
        self.module_hooks: dict[str, Any] = {}     # name -> holder module with user forward hooks
        self.head_grad_tmp: torch.Tensor | None = None
        self._graphs: dict[tuple, dict] = {}       # (B, S, loss_scale, labels-alias) -> captured micro-step
        self.decode_state = None                   # generation's KV caches + decode graph (models/generation.py)
        self.assisted_state = None                 # assisted generation's verify buffers, draft caches + round graph
        self.beam_state = None                     # beam search's caches, chunk table, selection state + step graph
        self.score_state = None                    # scoring buffers (models/scoring.py)
        self.fp8_weights = None                    # e4m3 + dequantised projection weights of fp8_weights=True (models/fp8_weights.py)

    def workspace(self, B: int, S: int) -> _Workspace:
        key = (B, S, str(self.arena.device), self.arena.compute_dtype)
        ws = self._ws.get(key)
        if ws is None:
            if len(self._ws) >= 2:       # keep at most two shapes resident (train + eval)
                old = next(iter(self._ws))
                self._ws.pop(old)
                for gk in [k for k in self._graphs if k[:2] == old[:2]]:      # graphs captured on the evicted buffers
                    del self._graphs[gk]
            if self.fp8 and self.arena.device.type == "cuda":
                F.check_tokens(B * S)
            ws = _Workspace(self.cfg, B, S, self.arena.device, self.arena.compute_dtype, self.lce_chunk)
            if self.fp8:
                ws.fp8 = _Fp8Workspace(self.cfg, B * S, self.arena.device)
            self._ws[key] = ws
        return ws

    # --------------------------------------------------------------------------------------------- forward
    def _fire_hooks(self, name: str, out: torch.Tensor) -> None:
        mod = self.module_hooks.get(name)
        if mod is not None and mod._forward_hooks:
            for hook in list(mod._forward_hooks.values()):
                hook(mod, (), out)

    def forward_hidden(self, ws: _Workspace, ids: torch.Tensor, attention_mask: torch.Tensor | None = None) -> torch.Tensor:
        cfg, ar = self.cfg, self.arena
        B, S, L = ws.B, ws.S, cfg.num_hidden_layers
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        f8 = ws.fp8
        ws.ids.copy_(ids.reshape(-1), non_blocking=True)
        K.embedding_fwd(ws.ids, ar.w("model.embed_tokens.weight"), out=ws.xa[0])
        delta = None
        for l in range(L):
            p = f"model.layers.{l}."
            x_prev = ws.xa[l] if l == 0 else ws.xm[l - 1]
            # --- attention block:  xa = x_prev + delta ; xn1 = norm(xa)
            K.rmsnorm_fwd(x_prev, ar.w(p + "input_layernorm.weight"), cfg.rms_norm_eps, delta=delta, out=ws.xn1[l],
                          rstd=ws.rstd1[l], x_out=ws.xa[l])
            if f8 is not None:
                xq, ix = f8.act(l, _F8_QKV, ws.xn1[l], f8.xn1_t[l])
                wq, iw = f8.weight(l, _F8_QKV, ar.qkv_w(l))
                F.linear_qkv_rope(xq, wq, ix, iw, ws.qkv[l], ws.cos, ws.sin, S, Hq + Hkv, D)
            elif D == 64 and TC.usable(ws.xn1[l], ar.qkv_w(l)):
                # wgmma GEMM with the rotary embedding applied in the epilogue (no separate RoPE pass over q|k)
                TC.linear_qkv_rope(ws.xn1[l], ar.qkv_w(l), ws.qkv[l], ws.cos, ws.sin, S, (Hq + Hkv) * D)
            else:
                G.mm_nt(ws.xn1[l], ar.qkv_w(l), out=ws.qkv[l])
                K.rope_(ws.qkv[l], ws.cos, ws.sin, S, Hq + Hkv, D)
            if attention_mask is None:
                ws.att[l], ws.aux[l] = A.attention_fwd(ws.qkv[l], B, S, Hq, Hkv, D)
            else:
                ws.att[l], ws.aux[l] = _masked_attention_fwd(ws.qkv[l], attention_mask, B, S, Hq, Hkv, D)
            if f8 is not None:
                xq, ix = f8.act(l, _F8_O, ws.att[l], f8.att_t[l])
                wq, iw = f8.weight(l, _F8_O, ar.w(p + "self_attn.o_proj.weight"))
                F.linear(xq, wq, ix, iw, out=ws.proj)
            else:
                G.mm_nt(ws.att[l], ar.w(p + "self_attn.o_proj.weight"), out=ws.proj)
            if self.collect_act_norms:
                self.act_norms[f"activation/{p}self_attn"] = ws.proj.float().norm(p=2)
            self._fire_hooks(p + "self_attn", ws.proj)
            # --- MLP block:  xm = xa + proj ; xn2 = norm(xm)
            K.rmsnorm_fwd(ws.xa[l], ar.w(p + "post_attention_layernorm.weight"), cfg.rms_norm_eps, delta=ws.proj,
                          out=ws.xn2[l], rstd=ws.rstd2[l], x_out=ws.xm[l])
            if f8 is not None:
                xq, ix = f8.act(l, _F8_GU, ws.xn2[l], f8.xn2_t[l])
                wq, iw = f8.weight(l, _F8_GU, ar.gu_w(l))
                F.linear_swiglu(xq, wq, ix, iw, ws.gu[l], ws.act[l])
                xq, ix = f8.act(l, _F8_DOWN, ws.act[l], f8.act_t[l])
                wq, iw = f8.weight(l, _F8_DOWN, ar.w(p + "mlp.down_proj.weight"))
                F.linear(xq, wq, ix, iw, out=ws.proj)
            else:
                if cfg.intermediate_size % 64 == 0 and TC.usable(ws.xn2[l], ar.gu_w(l)):
                    TC.linear_swiglu(ws.xn2[l], ar.gu_w(l), ws.gu[l], ws.act[l])     # SwiGLU is the GEMM epilogue
                else:
                    G.mm_nt(ws.xn2[l], ar.gu_w(l), out=ws.gu[l])
                    K.swiglu_fwd(ws.gu[l], out=ws.act[l])
                G.mm_nt(ws.act[l], ar.w(p + "mlp.down_proj.weight"), out=ws.proj)
            delta = ws.proj
        K.rmsnorm_fwd(ws.xm[L - 1], ar.w("model.norm.weight"), cfg.rms_norm_eps, delta=delta, out=ws.xnf, rstd=ws.rstdf,
                      x_out=ws.xf)
        return ws.xnf

    # --------------------------------------------------------------------------------------------- LM head + loss
    def head_loss(self, ws: _Workspace, labels: torch.Tensor | None, loss_scale: float, with_grad: bool,
                  direct: bool) -> torch.Tensor:
        """Linear-cross-entropy of the LM head.  Returns the mean loss (0-dim fp32 tensor on device).

        with_grad: also produce d(xnf) in ws.dxnf and the lm_head weight gradient, scaled by loss_scale / n_valid.
        direct: accumulate the lm_head gradient into the arena now (scale known); otherwise into ``head_grad_tmp`` so
        that autograd can apply the upstream gradient later.

        CUDA bf16: the fused path (``_head_loss_fused``) - logits never exist.  Other dtypes / CPU: the reference path
        that materialises a logits tile per chunk (same math, PyTorch ops).
        Reference call site: train_diloco_torch.py:313-314 / train_fsdp.py:378-379 -> loss_utils.py:45-67.
        """
        cfg, ar = self.cfg, self.arena
        V = cfg.vocab_size
        # HF shift: position s predicts token s+1 ; last position of every sequence is ignored
        src = labels.reshape(-1)
        if src.device != ws.labels.device or src.dtype != torch.int64 or not src.is_contiguous():
            ws.labels_in.copy_(src, non_blocking=True)
            src = ws.labels_in
        K.lce_prep(src, ws.labels, ws.B, ws.S, loss_scale, ws.n_valid, ws.gscale, ws.loss_sum)
        w_lm = ar.w("lm_head.weight")
        hooked = self.module_hooks.get("lm_head")
        want_norm = self.collect_act_norms or (hooked is not None and bool(hooked._forward_hooks))
        if want_norm:
            ws.sumsq.zero_()
        g_lm = None
        if with_grad:
            if direct:
                g_lm = ar.g("lm_head.weight")
            else:
                if self.head_grad_tmp is None:
                    self.head_grad_tmp = torch.zeros(V, cfg.hidden_size, dtype=torch.float32, device=ar.device)
                else:
                    self.head_grad_tmp.zero_()
                g_lm = self.head_grad_tmp
        if TC.lce_usable(ws.xnf, w_lm) and os.environ.get("ODB_LCE_FUSED", "1") != "0":
            self._head_loss_fused(ws, w_lm, g_lm, want_norm)
        else:
            self._head_loss_reference(ws, w_lm, g_lm, want_norm)
        if want_norm:
            nrm = ws.sumsq.sqrt()[0]
            if self.collect_act_norms:
                self.act_norms["activation/lm_head"] = nrm
            if hooked is not None and hooked._forward_hooks:
                self._fire_hooks("lm_head", _NormOnly(nrm))
        return (ws.loss_sum / ws.n_valid)[0]

    def _head_loss_fused(self, ws: _Workspace, w_lm: torch.Tensor, g_lm: torch.Tensor | None, want_norm: bool) -> None:
        """Fused linear-cross-entropy on the wgmma GEMM (SURVEY K7).  Per chunk of rows:

          c_t   = x_t . W[y_t] + 58 ln 2                     (lce_label_dot: the label logit, 2 x T x h bytes)
          E     = exp(X W^T - c)   + partial row sums        (ONE GEMM, epilogue in registers; bf16 E only when training)
          S_t, loss_t = log S_t + 58 ln 2, rowscale_t = gscale / S_t, xs = rowscale * x, dW[y_t] -= gscale x_t  (lce_finalize)
          dX    = rowscale * (E W) - gscale W[y]             (dgrad GEMM, W read MN-major, normaliser + one-hot in the epilogue)
          dW   += E^T xs                                     (weight-gradient GEMM)

        softmax - onehot is never formed and there is no pass over a [T, V] tensor outside the three GEMMs: the shift c is
        known before the GEMM, so the exponentials can be emitted by its epilogue, and the per-row normaliser moves to
        the fp32 side of the two gradient GEMMs.  In evaluation (g_lm is None) nothing of size [T, V] is written at all.
        The shift puts the label's exponential at exactly 2^-58 (a bf16 value), so rowscale * E_y - gscale is gscale (p_y - 1)
        without a rounding bias even for a confidently predicted label (tests/test_loss_head_oracle_gpu.py).
        """
        T, h = ws.T, self.cfg.hidden_size
        V = w_lm.shape[0]
        planes = TC.lce_planes(V)
        shift, rowscale, partials, e_buf, xs_buf = ws.lce_buffers(planes, h)
        train = g_lm is not None
        K.lce_label_dot(ws.xnf, w_lm, ws.labels, shift)
        C = ws.lce_rows
        for c0 in range(0, T, C):
            c1 = min(T, c0 + C)
            n = c1 - c0
            x = ws.xnf[c0:c1]
            e = e_buf[:n] if train else None
            TC.lce_fwd(x, w_lm, shift[c0:c1], partials, e, want_sumsq=want_norm)
            K.lce_finalize(partials, planes, ws.labels[c0:c1], ws.gscale, ws.loss_sum, ws.sumsq if want_norm else None,
                           rowscale[c0:c1] if train else None, x, xs_buf[:n] if train else None, g_lm)
            if train:
                TC.lce_dx(e, w_lm, rowscale[c0:c1], ws.labels[c0:c1], ws.gscale, ws.dxnf[c0:c1])
                G.mm_tn_acc(e, xs_buf[:n], g_lm)

    def _head_loss_reference(self, ws: _Workspace, w_lm: torch.Tensor, g_lm: torch.Tensor | None, want_norm: bool) -> None:
        T = ws.T
        C = ws.lce_rows
        for c0 in range(0, T, C):
            c1 = min(T, c0 + C)
            logits = ws.logits[: c1 - c0]
            G.mm_nt(ws.xnf[c0:c1], w_lm, out=logits)
            if g_lm is not None:
                K.ce_fwd_bwd_(logits, ws.labels[c0:c1], ws.gscale, ws.loss_sum, ws.sumsq if want_norm else None)
                G.mm_nn(logits, w_lm, out=ws.dxnf[c0:c1])
                G.mm_tn_acc(logits, ws.xnf[c0:c1], g_lm)
            else:
                if want_norm:
                    ws.sumsq.add_(logits.float().pow(2).sum())
                K.ce_fwd(logits, ws.labels[c0:c1], ws.loss_sum)

    def logits(self, ws: _Workspace) -> torch.Tensor:
        """Materialise full logits [T, V] (inference / debugging only)."""
        return G.mm_nt(ws.xnf, self.arena.w("lm_head.weight"))

    # --------------------------------------------------------------------------------------------- backward
    def backward(self, ws: _Workspace, attention_mask: torch.Tensor | None = None) -> None:
        """Back-propagate ws.dxnf (gradient w.r.t. the final-norm output) through the stack, accumulating into arena.grad."""
        cfg, ar = self.cfg, self.arena
        B, S, L = ws.B, ws.S, cfg.num_hidden_layers
        Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        f8 = ws.fp8
        K.rmsnorm_bwd(ws.dxnf, ws.xf, ar.w("model.norm.weight"), ws.rstdf, None, ws.dx, ar.g("model.norm.weight"))
        for l in reversed(range(L)):
            p = f"model.layers.{l}."
            # ---- MLP block (ws.dx is the gradient of x_out = xm + down(act))
            w_down = ar.w(p + "mlp.down_proj.weight")
            if f8 is not None:
                gq, gt, ig = f8.grad(l, _F8_DOWN, ws.dx)
                F.wgrad(gt, f8.act_t[l], ig, f8.act_inv(l, _F8_DOWN), ar.g(p + "mlp.down_proj.weight"))
                wt, iw = f8.weight_t(l, _F8_DOWN, w_down)
                F.linear_swiglu_bwd(gq, wt, ig, iw, ws.gu[l])
                gq, gt, ig = f8.grad(l, _F8_GU, ws.gu[l])
                F.wgrad(gt, f8.xn2_t[l], ig, f8.act_inv(l, _F8_GU), ar.gu_g(l))
                wt, iw = f8.weight_t(l, _F8_GU, ar.gu_w(l))
                F.linear(gq, wt, ig, iw, out=ws.dn)
            else:
                G.mm_tn_acc(ws.dx, ws.act[l], ar.g(p + "mlp.down_proj.weight"))
                if TC.swiglu_bwd_usable(ws.dx, w_down, ws.gu[l]):
                    TC.linear_swiglu_bwd(ws.dx, w_down, ws.gu[l])              # dgrad GEMM with the SwiGLU backward as epilogue
                else:
                    G.mm_nn(ws.dx, w_down, out=ws.dact)
                    K.swiglu_bwd(ws.dact, ws.gu[l], ws.gu[l])                  # in place: gu <- d(gu)
                G.mm_tn_acc(ws.gu[l], ws.xn2[l], ar.gu_g(l))
                G.mm_nn(ws.gu[l], ar.gu_w(l), out=ws.dn)
            K.rmsnorm_bwd(ws.dn, ws.xm[l], ar.w(p + "post_attention_layernorm.weight"), ws.rstd2[l], ws.dx, ws.dx,
                          ar.g(p + "post_attention_layernorm.weight"))
            # ---- attention block (ws.dx is now the gradient of xm = xa + o(att))
            if f8 is not None:
                gq, gt, ig = f8.grad(l, _F8_O, ws.dx)
                F.wgrad(gt, f8.att_t[l], ig, f8.act_inv(l, _F8_O), ar.g(p + "self_attn.o_proj.weight"))
                wt, iw = f8.weight_t(l, _F8_O, ar.w(p + "self_attn.o_proj.weight"))
                F.linear(gq, wt, ig, iw, out=ws.datt)
            else:
                G.mm_tn_acc(ws.dx, ws.att[l], ar.g(p + "self_attn.o_proj.weight"))
                G.mm_nn(ws.dx, ar.w(p + "self_attn.o_proj.weight"), out=ws.datt)
            parts_ok = (f8 is None and attention_mask is None and cfg.q_dim % 64 == 0 and cfg.kv_dim % 64 == 0
                        and TC.nn_usable(ws.datt, ar.qkv_w(l)))
            if attention_mask is None:
                res = A.attention_bwd(ws.datt, ws.qkv[l], ws.att[l], ws.aux[l], ws.dqkv, B, S, Hq, Hkv, D, want_parts=parts_ok,
                                      rope=(ws.cos, ws.sin))
            else:
                _masked_attention_bwd(ws.datt, ws.aux[l], ws.dqkv, B, S, Hq, Hkv, D)
                res = ws.dqkv
            if isinstance(res, tuple):
                # un-packed gradients (cuDNN): rotate dq/dk in place, three wgrads into the row blocks of the fused
                # QKV gradient, and ONE dgrad GEMM whose A operand is read from the three tensors
                dq, dk, dv = res
                K.rope_(dq, ws.cos, ws.sin, S, Hq, D, backward=True)
                K.rope_(dk, ws.cos, ws.sin, S, Hkv, D, backward=True)
                gq = ar.qkv_g(l)
                if cfg.q_dim % 256 == 0 and cfg.kv_dim % 256 == 0 and TC.wgrad_usable(dq, dk, dv, ws.xn1[l]):
                    TC.wgrad_acc((dq, dk, dv), ws.xn1[l], gq)          # one launch, A read from the three tensors
                else:
                    G.mm_tn_acc(dq, ws.xn1[l], gq[: cfg.q_dim])
                    G.mm_tn_acc(dk, ws.xn1[l], gq[cfg.q_dim: cfg.q_dim + cfg.kv_dim])
                    G.mm_tn_acc(dv, ws.xn1[l], gq[cfg.q_dim + cfg.kv_dim:])
                TC.linear_nn_a3(dq, dk, dv, ar.qkv_w(l), ws.dn)
            else:
                if attention_mask is not None or not A.bwd_applies_rope(ws.aux[l]):
                    K.rope_(ws.dqkv, ws.cos, ws.sin, S, Hq + Hkv, D, backward=True)
                if f8 is not None:
                    gq, gt, ig = f8.grad(l, _F8_QKV, ws.dqkv)
                    F.wgrad(gt, f8.xn1_t[l], ig, f8.act_inv(l, _F8_QKV), ar.qkv_g(l))
                    wt, iw = f8.weight_t(l, _F8_QKV, ar.qkv_w(l))
                    F.linear(gq, wt, ig, iw, out=ws.dn)
                else:
                    G.mm_tn_acc(ws.dqkv, ws.xn1[l], ar.qkv_g(l))
                    G.mm_nn(ws.dqkv, ar.qkv_w(l), out=ws.dn)
            K.rmsnorm_bwd(ws.dn, ws.xa[l], ar.w(p + "input_layernorm.weight"), ws.rstd1[l], ws.dx, ws.dx,
                          ar.g(p + "input_layernorm.weight"))
            ws.att[l] = None
            ws.aux[l] = None
        K.embedding_bwd(ws.ids, ws.dx, ar.g("model.embed_tokens.weight"))

    # --------------------------------------------------------------------------------------------- fused entry
    def forward_backward(self, ids: torch.Tensor, labels: torch.Tensor, loss_scale: float = 1.0,
                         attention_mask: torch.Tensor | None = None) -> torch.Tensor:
        """One micro-batch: forward, loss, backward; gradients (scaled by loss_scale) are ADDED to arena.grad.
        Returns the mean token loss as a device scalar (no host sync)."""
        B, S = ids.shape
        ws = self.workspace(B, S)
        mask = _normalize_mask(attention_mask)
        ar = self.arena
        with torch.no_grad():
            ar.materialize_shadow()            # FULL_SHARD: all-gather the compute weights (no-op otherwise)
            self.forward_hidden(ws, ids, mask)
            loss = self.head_loss(ws, labels, loss_scale, with_grad=True, direct=True)
            if ar.param_sharded:               # reshard after forward, gather again for backward (FSDP FULL_SHARD)
                ar.release_shadow()
                ar.materialize_shadow()
            self.backward(ws, mask)
            ar.release_shadow()
        return loss


    # --------------------------------------------------------------------------------------------- CUDA-graph replay
    def forward_backward_graphed(self, ids: torch.Tensor, labels: torch.Tensor, loss_scale: float) -> torch.Tensor:
        """``forward_backward`` with the ~250 launches of a micro-batch captured ONCE per (B, S, loss_scale) into a CUDA
        graph and replayed afterwards (every buffer of the micro-step is static: workspace, arena, TMA descriptors are
        baked kernel parameters).  Inputs are copied into the graph's static id / label buffers; the returned loss is the
        graph's static output (consume it before the next replay).  Falls back to the eager path while hooks /
        activation-norm collection are active (they run Python between kernels)."""
        B, S = ids.shape
        hooked = any(m._forward_hooks for m in self.module_hooks.values())
        if self.collect_act_norms or hooked or not ids.is_cuda:
            return self.forward_backward(ids, labels, loss_scale)
        key = (B, S, float(loss_scale), labels is ids)
        st = self._graphs.get(key)
        if st is not None and st.get("version") != self.arena.version:
            st = None                     # an arena buffer was re-homed (symmetric-memory windows): captured pointers are stale
        if st is None:
            st = {"calls": 0, "graph": None, "version": self.arena.version}
            self._graphs[key] = st
        if st["graph"] is None:
            st["calls"] += 1
            if st["calls"] <= 2:          # warm-up: allocations, cudaFuncSetAttribute, library handles
                return self.forward_backward(ids, labels, loss_scale)
            g_ids = torch.empty_like(ids)
            g_lab = g_ids if labels is ids else torch.empty_like(labels)
            g_ids.copy_(ids)
            if g_lab is not g_ids:
                g_lab.copy_(labels)
            ws = self.workspace(B, S)
            for l in range(self.cfg.num_hidden_layers):
                ws.att[l] = ws.aux[l] = None
            torch.cuda.synchronize(ids.device)
            graph = torch.cuda.CUDAGraph()
            n0 = _lib.launch_count()
            # thread_local: the NCCL watchdog / data-loader threads keep making CUDA calls of their own during the capture
            with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                loss = self.forward_backward(g_ids, g_lab, loss_scale)
            # kernels of ours recorded in the graph: every replay launches them again (bench.py's gpu_launches book-keeping)
            st.update(graph=graph, ids=g_ids, labels=g_lab, loss=loss, kernels=_lib.launch_count() - n0)
            graph.replay()
            return st["loss"]
        st["ids"].copy_(ids, non_blocking=True)
        if st["labels"] is not st["ids"]:
            st["labels"].copy_(labels, non_blocking=True)
        st["graph"].replay()
        _lib.count_launch(st["kernels"])
        return st["loss"]


class _NormOnly:
    """Stand-in handed to lm_head forward hooks: the logits are never materialised, only their L2 norm exists."""

    def __init__(self, nrm: torch.Tensor):
        self._nrm = nrm

    def norm(self, p=2):
        return self._nrm


def _normalize_mask(attention_mask: torch.Tensor | None) -> torch.Tensor | None:
    """None when the mask is absent or all ones (pure causal fast path)."""
    if attention_mask is None:
        return None
    if bool(attention_mask.all()):
        return None
    return attention_mask.bool()


def _masked_attention_fwd(qkv, mask, B, S, Hq, Hkv, D):
    """Padding-mask path (real text with pad tokens): library SDPA with an explicit mask, differentiated by autograd."""
    q, k, v = A.split_qkv(qkv, B, S, Hq, Hkv, D)
    leaves = [t.detach().transpose(1, 2).requires_grad_(True) for t in (q, k, v)]
    causal = torch.ones(S, S, dtype=torch.bool, device=qkv.device).tril()
    full = causal[None, None] & mask[:, None, None, :].to(qkv.device)
    # keep fully-masked rows finite (pad queries): let them see themselves
    full = full | torch.eye(S, dtype=torch.bool, device=qkv.device)[None, None]
    with torch.enable_grad():
        o = torch.nn.functional.scaled_dot_product_attention(leaves[0], leaves[1], leaves[2], attn_mask=full,
                                                             enable_gqa=(Hq != Hkv))
        out = o.transpose(1, 2).reshape(B * S, Hq * D)
    return out.detach(), (out, leaves)


def _masked_attention_bwd(dout, aux, dqkv, B, S, Hq, Hkv, D):
    out, leaves = aux
    gq, gk, gv = torch.autograd.grad(out, leaves, dout)
    dq, dk, dv = A.split_qkv(dqkv, B, S, Hq, Hkv, D)
    dq.copy_(gq.transpose(1, 2))
    dk.copy_(gk.transpose(1, 2))
    dv.copy_(gv.transpose(1, 2))


# ======================================================================================================= nn.Module facade
class _Holder(nn.Module):
    """Parameter holder: the math runs in LlamaEngine, this only gives the weight its HF name."""

    def __init__(self, weight: nn.Parameter | None = None):
        super().__init__()
        if weight is not None:
            self.weight = weight

    def forward(self, *a, **k):  # pragma: no cover
        raise RuntimeError("sub-modules of opendiloco_b200.LlamaForCausalLM are parameter holders; call the top-level model")


class _EngineLoss(torch.autograd.Function):
    """Single autograd node bridging loss.backward() to the engine's hand-written backward."""

    @staticmethod
    def forward(ctx, anchor: torch.Tensor, model: "LlamaForCausalLM", ids, labels, mask):
        eng = model.engine
        B, S = ids.shape
        ws = eng.workspace(B, S)
        eng.arena.materialize_shadow()
        eng.forward_hidden(ws, ids, mask)
        loss = eng.head_loss(ws, labels, 1.0, with_grad=True, direct=False)
        eng.arena.release_shadow()
        ctx.model, ctx.ws, ctx.mask = model, ws, mask
        return loss.clone()

    @staticmethod
    def backward(ctx, g):
        eng, ws = ctx.model.engine, ctx.ws
        with torch.no_grad():
            g32 = g.to(torch.float32)
            ws.dxnf.mul_(g32.to(ws.dxnf.dtype))
            eng.arena.g("lm_head.weight").addcmul_(eng.head_grad_tmp, g32.expand_as(eng.head_grad_tmp))
            eng.arena.materialize_shadow()
            eng.backward(ws, ctx.mask)
            eng.arena.release_shadow()
        return None, None, None, None, None


class LlamaForCausalLM(nn.Module):
    """Drop-in for the HF class the reference trains (train_fsdp.py:171-174, train_diloco_torch.py:183)."""

    def __init__(self, config: LlamaConfig, device=None, precision: str = "bf16-mixed", seed: int | None = None,
                 init: bool = True, lce_chunk: int = 32768):
        """``precision``: "bf16-mixed", "fp16-mixed", "32-true" (compute weights and activations in that dtype, fp32 master
        weights and gradients), or "fp8-mixed": bf16-mixed with the q|k|v, o, gate|up and down projections of every decoder
        layer run as FP8 GEMMs in forward, dgrad and wgrad (e4m3 activations and weights, e5m2 gradients, per-tensor
        current scaling; see ops/fp8.py).  On CUDA, fp8-mixed raises ValueError for shapes the FP8 kernels do not cover."""
        super().__init__()
        self.config = config
        self.precision = precision
        compute = {"bf16-mixed": torch.bfloat16, "fp16-mixed": torch.float16, "32-true": torch.float32,
                   "fp8-mixed": torch.bfloat16}[precision]
        device = torch.device(device if device is not None else "cpu")
        if precision == "fp8-mixed" and device.type == "cuda":
            F.check_config(config)
        self.arena = ParamArena(config, device, compute)
        self.engine = LlamaEngine(config, self.arena, lce_chunk=lce_chunk, fp8=precision == "fp8-mixed")
        self._build_tree()
        if init:
            self.arena.init_weights(seed)

    # ------------------------------------------------------------------ module tree with HF names
    def _build_tree(self) -> None:
        cfg, ar = self.config, self.arena

        def P(name: str) -> nn.Parameter:
            prm = nn.Parameter(ar.p(name), requires_grad=True)
            prm.grad = ar.g(name)
            prm._odb_name = name
            prm._odb_arena = ar
            return prm

        self.model = _Holder()
        self.model.embed_tokens = _Holder(P("model.embed_tokens.weight"))
        layers = []
        for l in range(cfg.num_hidden_layers):
            p = f"model.layers.{l}."
            layer = _Holder()
            layer.self_attn = _Holder()
            for n in ("q_proj", "k_proj", "v_proj", "o_proj"):
                setattr(layer.self_attn, n, _Holder(P(p + f"self_attn.{n}.weight")))
            layer.mlp = _Holder()
            for n in ("gate_proj", "up_proj", "down_proj"):
                setattr(layer.mlp, n, _Holder(P(p + f"mlp.{n}.weight")))
            layer.input_layernorm = _Holder(P(p + "input_layernorm.weight"))
            layer.post_attention_layernorm = _Holder(P(p + "post_attention_layernorm.weight"))
            layers.append(layer)
            self.engine.module_hooks[p + "self_attn"] = layer.self_attn
        self.model.layers = nn.ModuleList(layers)
        self.model.norm = _Holder(P("model.norm.weight"))
        self.lm_head = _Holder(P("lm_head.weight"))
        self.engine.module_hooks["lm_head"] = self.lm_head

    def _rebind(self) -> None:
        for _, prm in self.named_parameters():
            prm.data = self.arena.p(prm._odb_name)
            prm.grad = self.arena.g(prm._odb_name)

    # ------------------------------------------------------------------ device / dtype management
    def to(self, *args, **kwargs):
        device = kwargs.get("device")
        for a in args:
            if isinstance(a, (str, torch.device, int)):
                device = a
            elif isinstance(a, torch.dtype):
                raise TypeError("opendiloco_b200 models keep fp32 master weights; choose `precision=` at construction")
        if device is not None:
            device = torch.device("cuda", device) if isinstance(device, int) else torch.device(device)
            if device.type == "cuda" and device.index is None:
                device = torch.device("cuda", torch.cuda.current_device())
            if device != self.arena.device:
                if self.engine.fp8 and device.type == "cuda":
                    F.check_config(self.config)
                self.arena.migrate(device)
                self.engine._ws.clear()
                self.engine._graphs.clear()
                self.engine.decode_state = None
                self.engine.assisted_state = None
                self.engine.beam_state = None
                self.engine.score_state = None
                self.engine.fp8_weights = None
                self.engine.head_grad_tmp = None
                self._rebind()
        return self

    def cuda(self, device=None):
        return self.to(torch.device("cuda", device if device is not None else torch.cuda.current_device()))

    def cpu(self):
        return self.to("cpu")

    @property
    def device(self) -> torch.device:
        return self.arena.device

    # ------------------------------------------------------------------ forward
    def forward(self, input_ids: torch.Tensor, attention_mask: torch.Tensor | None = None,
                labels: torch.Tensor | None = None, return_logits: bool = False, **_unused) -> CausalLMOutput:
        eng = self.engine
        if input_ids.device != self.arena.device:
            input_ids = input_ids.to(self.arena.device, non_blocking=True)
        if labels is not None and labels.device != self.arena.device:
            labels = labels.to(self.arena.device, non_blocking=True)
        mask = _normalize_mask(attention_mask)
        B, S = input_ids.shape
        if labels is not None and torch.is_grad_enabled() and self.training:
            loss = _EngineLoss.apply(self.lm_head.weight, self, input_ids, labels, mask)
            return CausalLMOutput(loss=loss)
        with torch.no_grad():
            ws = eng.workspace(B, S)
            self.arena.materialize_shadow()
            eng.forward_hidden(ws, input_ids, mask)
            loss = eng.head_loss(ws, labels, 1.0, with_grad=False, direct=False).clone() if labels is not None else None
            logits = eng.logits(ws).view(B, S, -1) if (return_logits or labels is None) else None
            self.arena.release_shadow()
        return CausalLMOutput(loss=loss, logits=logits)

    def forward_backward(self, input_ids: torch.Tensor, labels: torch.Tensor, loss_scale: float = 1.0,
                         attention_mask: torch.Tensor | None = None) -> torch.Tensor:
        """Native fast path: one micro-batch forward+backward, grads += loss_scale * dL/dw. Returns the device loss.
        With ODB_CUDA_GRAPH=1 (and no padding mask) the micro-step is replayed from a CUDA graph."""
        if (_use_graph() and attention_mask is None and input_ids.is_cuda and self.arena.compute_dtype == torch.bfloat16
                and not self.arena.param_sharded):
            return self.engine.forward_backward_graphed(input_ids, labels, loss_scale)
        return self.engine.forward_backward(input_ids, labels, loss_scale, attention_mask)

    @torch.no_grad()
    def generate(self, input_ids: torch.Tensor, attention_mask: torch.Tensor | None = None, max_new_tokens: int = 20,
                 do_sample: bool = False, temperature: float = 1.0, top_k: int = 50, top_p: float = 1.0, eos_token_id=None,
                 pad_token_id: int | None = None, seed: int = 0, assistant_model: "LlamaForCausalLM | None" = None,
                 num_assistant_tokens: int = 4, num_beams: int = 1, length_penalty: float = 1.0, early_stopping=False,
                 num_return_sequences: int = 1, return_dict_in_generate: bool = False, repetition_penalty: float = 1.0,
                 no_repeat_ngram_size: int = 0, min_new_tokens: int = 0, prompt_lookup_num_tokens: int | None = None,
                 max_matching_ngram_size: int | None = None, fp8_weights: bool = False, fp8_kv_cache: bool = False,
                 sequence_bias=None, bad_words_ids=None, min_length: int = 0, min_p: float | None = None,
                 output_scores: bool = False, output_logits: bool = False):
        """KV-cached text generation with HF ``generate`` keyword names.  Returns LongTensor [B, P + max_new_tokens]: the
        prompt as given, then the new tokens.

        Prompts may be left-padded with an ``attention_mask``.  ``do_sample=False`` is greedy (ties to the lowest id);
        otherwise temperature, top-k (0 = off), top-p and ``min_p`` (in [0, 1]; None or 0 is off: keep the tokens whose
        probability is at least min_p times the largest) are applied in HF's order and tokens are drawn with ``seed``.
        ``min_p`` is a warper, so it does nothing without ``do_sample`` (greedy, beam search) and works with
        ``assistant_model`` and ``prompt_lookup_num_tokens``, whose acceptance applies it to both distributions.
        ``eos_token_id`` (int or list) defaults to ``config.eos_token_id``; after a row emits it, the row is filled with
        ``pad_token_id`` (default: the first EOS id).  Reads the current compute weights.  bf16-mixed CUDA models run the
        decode kernels (csrc/decode_sm90.cu) with the step replayed from a CUDA graph; other precisions and devices run the
        PyTorch reference path.  fp8-mixed models generate on the bf16 path from their bf16 compute weights (no FP8 GEMMs).
        Raises ValueError for a parameter-sharded (FULL_SHARD) model, a prompt plus
        ``max_new_tokens`` longer than ``max_position_embeddings``, or a mask that is not left-padded.

        ``assistant_model`` (a smaller model with the same vocabulary, on the same device and compute dtype; the model
        itself works too) turns on assisted (speculative) generation: each round the assistant proposes
        ``num_assistant_tokens`` (1..7) tokens, this model scores them all in one pass, and speculative sampling keeps
        an exact sample of this model's distribution (greedy: exactly its argmax continuation, up to bf16 near-ties
        between the one- and multi-token attention).  ``engine.assisted_state`` then reports ``verify_passes()`` and
        ``acceptance_rate()``.  Raises ValueError for a different vocabulary, device or compute dtype, a parameter-sharded
        assistant, ``num_assistant_tokens`` outside [1, 7], or a prompt plus ``max_new_tokens`` plus
        ``num_assistant_tokens`` beyond either model's ``max_position_embeddings``.

        ``prompt_lookup_num_tokens`` K (1..7; None is off) turns on prompt lookup decoding, transformers' draft-free
        speculative generation: each round, every row proposes up to K tokens from its own history (its real prompt tokens,
        then its generated ones; padding is not history), this model scores them in one pass and the same acceptance as
        assisted generation keeps an exact sample of its distribution (greedy: its argmax continuation, up to the same
        bf16 near-ties).  A row's proposals are the tokens that followed the earliest earlier occurrence of its last n
        tokens, for the largest n <= ``max_matching_ngram_size`` (1..64, default 2) that has one, at most K and cut before
        the first EOS id; a row with no match proposes nothing and gains one token that round.  ``engine.assisted_state``
        then reports ``verify_passes()`` and ``acceptance_rate()`` (accepted over proposed tokens).  Works with greedy
        decoding and sampling, left-padded batches and EOS.  Raises ValueError for K or ``max_matching_ngram_size`` outside
        those ranges or not an integer, together with ``assistant_model``, ``num_beams`` > 1 or any logits processor below
        (not supported yet), or for a prompt plus ``max_new_tokens`` plus K beyond ``max_position_embeddings``.

        ``num_beams`` > 1 (at most 8) runs deterministic beam search as transformers' ``generate(num_beams=...,
        do_sample=False)``: fp32 log-softmax of the logits, then the logits processors below, ``length_penalty``,
        ``early_stopping`` (True, False or ``"never"``) and the finished-hypothesis rules of HF, ties to the lower
        ``beam * V + token``.  It returns ``[B * num_return_sequences, P + max_new_tokens]``: row ``b * R + r`` is prompt b
        as given, then its r-th best hypothesis (EOS included), then ``pad_token_id``.  bf16-mixed CUDA models run the
        selection and cache-reorder kernels with each step replayed from a CUDA graph; beams share the complete 128-position
        cache chunks of their history through a chunk table.  Those kernels take num_beams * ceil(vocab_size / 1024) <= 512
        and at most 32768 positions; beyond that the step runs on the PyTorch references without a graph, with a warning.
        Raises ValueError for ``num_beams`` outside [1, 8],
        ``num_return_sequences`` outside [1, num_beams] with ``num_beams`` > 1, an unknown ``early_stopping``, or
        ``do_sample=True`` or ``assistant_model`` with ``num_beams`` > 1.

        Logits processors, HF's, applied in HF's order to the fp32 value of each logit (greedy and sampling: before the
        temperature, top-k, top-p and min-p warpers) or log-prob (beam search), on greedy, sampling and beam search:
        ``sequence_bias`` (HF's dict ``{tuple(ids): bias}`` or list ``[[ids], bias]``) adds a bias to the last token of a
        sequence: always for one id, and for a longer sequence when the history ends with its other ids (and is at least
        as long as the sequence); biases of one token are summed in HF's order (the length-1 one first, then dict order);
        ``repetition_penalty`` (a finite float > 0; 1.0 is off) then divides the positive and multiplies the negative values
        of every token in the row's history, once per distinct token; ``no_repeat_ngram_size`` n (0..64; 0 is off) forbids
        any n-gram from occurring twice in the history; ``bad_words_ids`` (a list of id lists) forbids the last id of each
        sequence by the matching rule of ``sequence_bias`` (single ids equal to an EOS id are dropped, as in HF);
        ``min_length`` (0 is off) forbids every EOS id while the history (prompt included) is shorter than it;
        ``min_new_tokens`` (0 is off) forbids every EOS id until that many tokens have been generated (nothing without EOS
        ids).  Sequences have 1..64 ids in [0, vocab_size); ``sequence_bias`` and ``bad_words_ids`` hold at most 1024
        sequences and 16384 ids together, and a bias may be -inf (a ban) but not NaN or +inf.  A row's history is its real prompt tokens followed by its
        generated tokens (beam search: the beam's own running sequence).  Unlike HF, the padding of a left-padded batch is
        not part of the history, so every row generates what it would alone.  A greedy row whose values are all -inf
        emits token 0; a sampled one its processed argmax.  With beam search, ``sequences_scores`` sum the processed
        log-probs, as in HF.  The settings live in device memory (the sequences in a fixed-capacity table): changing them
        replays the same CUDA graphs.  Raises ValueError for values outside those ranges, or for any of them on together
        with ``assistant_model`` or ``prompt_lookup_num_tokens`` (not supported yet).

        ``num_return_sequences`` n > 1 with ``do_sample=True`` and ``num_beams == 1`` draws n independent samples per
        prompt: ``[B * n, P + max_new_tokens]``, row ``b * n + j`` is prompt b as given, then its j-th sample; token for
        token what ``generate(input_ids.repeat_interleave(n, 0), attention_mask=attention_mask.repeat_interleave(n, 0),
        ...)`` returns with the same other arguments.  Each prompt is prefilled once; the n rows share its complete
        128-position cache chunks through a chunk table, and bf16-mixed CUDA models decode them on an sm_90a attention
        that loads a shared chunk once for several rows (the cache still holds B * n rows).  Works with the warpers, EOS,
        the logits processors, ``fp8_weights`` and ``fp8_kv_cache``.  Raises ValueError for n > 1 with
        ``do_sample=False`` and ``num_beams == 1``, or together with ``assistant_model`` or ``prompt_lookup_num_tokens``,
        and for an n that is not an integer >= 1.

        ``return_dict_in_generate=True`` returns a ``GenerateOutput`` with ``sequences`` and ``sequences_scores`` (fp32
        [B * num_return_sequences]: each hypothesis's summed log-probabilities / generated_len ** length_penalty; None
        without beam search).

        ``output_scores=True`` / ``output_logits=True`` (bools; ignored without ``return_dict_in_generate``, as in HF) add
        ``scores`` / ``logits`` to it: tuples of ``max_new_tokens`` fp32 tensors ``[rows, vocab_size]``, one per generated
        position, and with beam search ``beam_indices`` (int64 [B * num_return_sequences, max_new_tokens]: the running row
        ``b * num_beams + j`` that emitted each token of the hypothesis, -1 after it ends).  ``logits`` are the raw logits
        (the compute dtype's values, exactly).  ``scores`` follow HF per mode: greedy, the processed logits the argmax is
        taken of (the logits processors applied, bans as -inf); sampling and multi-sample, those divided by ``temperature``
        with -inf outside the set the token is drawn from (top-k, top-p and min-p; ``top_k=1`` keeps the argmax alone); beam
        search, the processed log_softmax of every running beam row (B * num_beams rows, in that step's order, without the
        running score); assisted and prompt lookup decoding, the target's processed and warped row of the slot that
        emitted each token.  ``compute_transition_scores`` turns them into per-token scores.  One deviation from HF: a
        column where a row (beam search: a prompt) had already finished holds a padding row, -inf everywhere and 0 at
        ``pad_token_id``, where HF keeps computing rows for finished sequences; so the tuples always have
        ``max_new_tokens`` entries and padding scores 0 in ``compute_transition_scores``.  The rows are written by the
        sm_90a sampler, acceptance and beam kernels into device buffers of rows * max_new_tokens * vocab_size * 6 bytes
        (about 790 MB at 8 rows, 512 tokens and 32000 ids), kept for the next call of the same shape; with both flags off
        nothing is allocated or launched for them.  Raises ValueError when either is not a bool.

        ``fp8_weights=True`` generates with FP8 weight-only quantisation: at the start of the call the q|k|v, o, gate|up
        and down projections of every decoder layer are quantised to e4m3 with one power-of-two scale per output row
        (ops/fp8w.py); the embedding, the norms and the LM head stay in the compute dtype.  The result is the model with
        every projection weight replaced by its dequantised copy Ŵ: bf16-mixed CUDA models decode on an sm_90a GEMM that
        streams the e4m3 weights (half the bytes of bf16) wherever a pass has at most 64 rows and run the bf16 GEMMs on Ŵ
        elsewhere (prefill, wider verify passes and beam steps); other precisions and devices run the reference path on
        Ŵ.  Works with every mode above; with ``assistant_model`` only this model is quantised.  While in use the e4m3 and
        dequantised copies take 1.5x the bf16 bytes of the projections (about 2.9 GB at the 1b preset), kept on the engine
        for the next call; training state is not touched.  Raises ValueError when ``fp8_weights`` is not a bool.

        ``fp8_kv_cache=True`` keeps the KV cache in FP8: every K/V row written into the decode cache (one (position, kv
        head) vector of ``head_dim`` values, the rotated k and the v the bf16 cache would store) is quantised to e4m3 with
        one power-of-two scale per row by the rule of ``fp8_weights`` (ops/fp8w.py ``quantize_rows_ref``; a non-finite row
        gives NaN bytes and factor), and stored as e4m3 [L, 2, B, Hkv, Smax, head_dim] plus an fp32 factor per row: 0.53x
        the bf16 cache bytes at head_dim 64.  The result is exactly this program with every cache write followed by
        replacing the written rows with their dequantised values q * inv: the prompt's own attention still reads its
        in-flight bf16 q|k|v (so the first new token is unchanged), and every later read (the one-token steps, the verify
        passes of assisted and prompt lookup decoding, beam steps, a token's own K/V included) sees the dequantised cache.
        Works with every mode above and together with ``fp8_weights``; with ``assistant_model`` only this model's cache
        is FP8.  ``False`` allocates and launches exactly what it did before.  Raises ValueError when ``fp8_kv_cache`` is
        not a bool."""
        from .generation import generate

        return generate(self, input_ids, attention_mask=attention_mask, max_new_tokens=max_new_tokens, do_sample=do_sample,
                        temperature=temperature, top_k=top_k, top_p=top_p, eos_token_id=eos_token_id, pad_token_id=pad_token_id,
                        seed=seed, assistant_model=assistant_model, num_assistant_tokens=num_assistant_tokens, num_beams=num_beams,
                        length_penalty=length_penalty, early_stopping=early_stopping, num_return_sequences=num_return_sequences,
                        return_dict_in_generate=return_dict_in_generate, repetition_penalty=repetition_penalty,
                        no_repeat_ngram_size=no_repeat_ngram_size, min_new_tokens=min_new_tokens,
                        prompt_lookup_num_tokens=prompt_lookup_num_tokens, max_matching_ngram_size=max_matching_ngram_size,
                        fp8_weights=fp8_weights, fp8_kv_cache=fp8_kv_cache, sequence_bias=sequence_bias,
                        bad_words_ids=bad_words_ids, min_length=min_length, min_p=min_p, output_scores=output_scores,
                        output_logits=output_logits)

    def compute_transition_scores(self, sequences: torch.Tensor, scores: tuple, beam_indices: torch.Tensor | None = None,
                                  normalize_logits: bool = False) -> torch.Tensor:
        """HF's ``compute_transition_scores``: the score of each generated token, [rows, generated length], from
        ``generate(..., return_dict_in_generate=True, output_scores=True)``'s ``sequences``, ``scores`` and (beam search)
        ``beam_indices``.  ``normalize_logits`` applies log_softmax to every score row first (per-token log-probabilities
        of sampled or greedy output).  Positions with a negative beam index score 0, and so do padding rows of finished
        sequences (their padding token has score 0).  Returns as many columns as the longest hypothesis (beam search) or
        ``len(scores)``.  The generated tokens are the last ``len(scores)`` columns of ``sequences``, as ``generate``
        returns them (always ``max_new_tokens`` wide); HF instead counts back from the end of sequences trimmed to the
        longest hypothesis, which would take the trailing padding here.  Plain torch on the scores' device."""
        V = self.config.vocab_size
        if beam_indices is None:
            beam_indices = torch.arange(scores[0].shape[0], device=sequences.device).view(-1, 1).expand(-1, len(scores))
        stacked = torch.stack(scores).reshape(len(scores), -1).transpose(0, 1)
        if normalize_logits:
            stacked = torch.log_softmax(stacked.reshape(-1, V, stacked.shape[-1]), dim=1).reshape(-1, stacked.shape[-1])
        mask = beam_indices < 0
        n = int((~mask).long().sum(-1).max())
        beam_indices = beam_indices.clone()[:, :n]
        mask = mask[:, :n]
        beam_indices[mask] = 0
        start = sequences.shape[-1] - len(scores)              # the first generated column
        idx = sequences[:, start:start + n].to(stacked.device) + beam_indices.to(stacked.device) * V
        out = stacked.gather(0, idx)
        out[mask.to(out.device)] = 0
        return out

    @torch.no_grad()
    def score(self, input_ids: torch.Tensor, attention_mask: torch.Tensor | None = None, labels: torch.Tensor | None = None,
              fp8_weights: bool = False):
        """Per-token log-likelihoods.  Returns ``ScoreOutput`` with ``logprobs`` (fp32 [B, S], log p(target_t | tokens < t))
        and ``greedy`` (bool [B, S], the argmax of the prediction at t-1, lowest index on ties, equals target_t), on the
        model's device.

        Targets follow HF ``labels``: entry t is about token t; ``labels`` (``-100`` = ignored) default to ``input_ids``.
        Position 0, padded and ignored positions give 0.0 / False.  ``attention_mask`` may hold any one contiguous run of
        ones per row (left, right or no padding); each row is scored like its unpadded tokens alone, positions from 0.
        Reads the current compute weights.  bf16-mixed CUDA models run the scoring LM-head kernels (no logits are written,
        exact for any logit range); other precisions and devices run the PyTorch reference path.  fp8-mixed models score on
        the bf16 path from their bf16 compute weights (no FP8 GEMMs), so their log-likelihoods differ slightly from the
        FP8 eval loss of ``forward``.  Raises ValueError for a
        parameter-sharded (FULL_SHARD) model, a sequence longer than ``max_position_embeddings``, mismatched shapes, a mask
        that is not one run per row, or token / label ids outside the vocabulary.

        ``fp8_weights=True`` scores the FP8 weight-only quantised model of ``generate(fp8_weights=True)`` (the projections
        replaced by their per-row e4m3 dequantised copies), which is how the quality cost of that quantisation is measured;
        a non-bool raises ValueError."""
        from .scoring import score

        return score(self, input_ids, attention_mask=attention_mask, labels=labels, fp8_weights=fp8_weights)

    # ------------------------------------------------------------------ state dict / checkpoints
    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        res = super().load_state_dict(state_dict, strict=strict, assign=False)
        self.arena.sync_shadow()
        return res

    def sync_compute_weights(self) -> None:
        """Call after writing to parameters outside the fused optimizers (torch optimizers, manual edits)."""
        self.arena.sync_shadow()

    @classmethod
    def from_config(cls, config: LlamaConfig, **kw) -> "LlamaForCausalLM":
        return cls(config, **kw)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path: str, config: LlamaConfig | None = None, device=None,
                        precision: str = "bf16-mixed", seed: int | None = 0, **_unused) -> "LlamaForCausalLM":
        """Load config (+ ``model.safetensors`` if present).  A bare config / preset name yields seeded random init —
        the offline equivalent of the reference's ``*-fresh`` hub checkpoints (init_weights.py:10-25)."""
        from ..utils.safetensors_io import load_safetensors

        cfg = config if isinstance(config, LlamaConfig) else LlamaConfig.from_pretrained(pretrained_model_name_or_path)
        path = Path(pretrained_model_name_or_path)
        st = path / "model.safetensors" if path.is_dir() else None
        model = cls(cfg, device=device, precision=precision, seed=seed, init=not (st and st.is_file()))
        if st is not None and st.is_file():
            tensors = load_safetensors(str(st))
            with torch.no_grad():
                for name in hf_param_order(cfg):
                    model.arena.p(name).copy_(tensors[name].to(torch.float32))
            model.arena.sync_shadow()
        return model

    def save_pretrained(self, directory: str) -> None:
        from ..utils.safetensors_io import save_safetensors

        os.makedirs(directory, exist_ok=True)
        self.config.save_pretrained(directory)
        save_safetensors({n: self.arena.p(n).detach().cpu().contiguous() for n in hf_param_order(self.config)},
                         os.path.join(directory, "model.safetensors"), metadata={"format": "pt"})

    def num_parameters(self) -> int:
        return self.config.num_parameters()

    @torch.no_grad()
    def clip_grad_norm_(self, max_norm: float, norm_type: float = 2.0) -> torch.Tensor:
        """FSDP-style method the reference calls (train_fsdp.py:395).  If a FusedAdamW owns the arena the scaling is
        folded into its next step (one reduction pass, zero extra sweeps); otherwise grads are scaled here."""
        assert norm_type == 2.0
        ref = getattr(self.arena, "fused_optimizer", None)
        opt = ref() if ref is not None else None
        if opt is not None:
            return opt.compute_grad_norm_partials(max_norm)
        total = self.arena.grad.norm(2)
        coef = torch.clamp(max_norm / (total + 1e-6), max=1.0)
        self.arena.grad.mul_(coef)
        return total
