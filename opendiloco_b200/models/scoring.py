"""Per-token log-likelihood scoring for :class:`~opendiloco_b200.models.llama.LlamaForCausalLM` (``model.score``).

Every row is compacted to start at position 0 and the batch is right-padded (to a multiple of 128 on the kernels), then
runs generation's layer program with prefill's attention (QKV(+RoPE) GEMM and the causal attention forward,
:func:`~opendiloco_b200.models.generation._prompt_attend`); causal attention keeps the right padding away from the real
positions.  The final-norm rows that predict a target are gathered
in output order and go through the LM head in chunks of at most ``SCORE_CHUNK`` rows:

    tc_gemm.lce_score           per 256-column plane: max, lowest argmax, sum exp(z - max), and the label logit
    kernels.lce_score_finalize  lse, logprob = z_label - lse, greedy = (argmax == label)

No logits are ever written, and the exponentials are taken relative to a maximum, so the log-probabilities are exact for
any logit range (the training LCE clamps its exponent).  CUDA bf16 models run the kernels of ``csrc/``; other precisions
and CPU models run the same program on the PyTorch references.

The buffers hang off the engine (one resident shape, like generation's decode state) and never go through
``LlamaEngine.workspace`` or its captured training graphs: scoring between training steps leaves them untouched.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

from ..ops import kernels as K
from ..ops import tc_gemm as TC
from . import fp8_weights as W8
from .generation import Rows, _layers, _prompt_attend, _resident, _round_up

SCORE_CHUNK = 32768                 # LM-head rows per scoring GEMM on the kernels
REFERENCE_CHUNK = 4096              # the reference materialises an fp32 [rows, V] logits chunk
IGNORE_INDEX = -100


@dataclass
class ScoreOutput:
    logprobs: torch.Tensor          # fp32 [B, S]: log p(target_t | tokens < t); 0 where nothing is scored
    greedy: torch.Tensor            # bool [B, S]: the prediction at t-1 (lowest-index argmax) equals target_t


class ScoreState:
    """Layer buffers for [B, Sp] compacted rows, the gathered LM-head rows of the B*S output slots and the plane
    statistics of one LM-head chunk."""

    def __init__(self, cfg, B: int, Sp: int, S: int, device, dtype, kernels: bool):
        n = B * S
        self.pb = Rows(cfg, B * Sp, device, dtype)
        self.cos, self.sin = K.rope_tables(Sp, cfg.head_dim, cfg.rope_theta, device)
        self.xg = torch.empty(n, cfg.hidden_size, dtype=dtype, device=device)
        self.gidx = torch.empty(n, dtype=torch.int64, device=device)
        self.labels = torch.empty(n, dtype=torch.int64, device=device)
        self.chunk = min(SCORE_CHUNK if kernels else REFERENCE_CHUNK, n)
        self.planes = (cfg.vocab_size + TC.SCORE_PLANE - 1) // TC.SCORE_PLANE
        f32 = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=device)  # noqa: E731
        self.pmax, self.psum, self.zlab = f32(self.planes * self.chunk), f32(self.planes * self.chunk), f32(self.chunk)
        self.pidx = torch.empty(self.planes * self.chunk, dtype=torch.int32, device=device)


def score_state(model, B: int, Sp: int, S: int, kernels: bool) -> ScoreState:
    """The model's scoring state for this shape, allocated on first use; at most one is resident."""
    ar = model.arena
    return _resident(model, "score_state", (B, Sp, S, str(ar.device), ar.compute_dtype, kernels),
                     lambda: ScoreState(model.config, B, Sp, S, ar.device, ar.compute_dtype, kernels))


def _plan(cfg, input_ids, attention_mask, labels, kernels: bool):
    """Host-side bookkeeping: validate the inputs and build (compacted ids [B, Sp], gather index [B*S], labels [B*S])."""
    if input_ids.dim() != 2:
        raise ValueError(f"input_ids must be [batch, length], got shape {tuple(input_ids.shape)}")
    B, S = input_ids.shape
    if B == 0 or S == 0:
        raise ValueError(f"input_ids is empty: shape {tuple(input_ids.shape)}")
    if S > cfg.max_position_embeddings:
        raise ValueError(f"sequence length {S} exceeds max_position_embeddings {cfg.max_position_embeddings}")
    ids = input_ids.detach().cpu().long()
    if attention_mask is None:
        lens = torch.full((B,), S, dtype=torch.int64)
        start = torch.zeros(B, dtype=torch.int64)
    else:
        if tuple(attention_mask.shape) != (B, S):
            raise ValueError(f"attention_mask shape {tuple(attention_mask.shape)} differs from input_ids {(B, S)}")
        m = attention_mask.detach().cpu().bool()
        runs = m[:, 0].long() + (m[:, 1:] & ~m[:, :-1]).sum(dim=1)
        if not bool((runs == 1).all()):
            raise ValueError("attention_mask must hold one contiguous run of ones in every row (left, right or no padding)")
        lens = m.sum(dim=1)
        start = m.long().argmax(dim=1)
    if labels is None:
        tgt = ids
    else:
        if tuple(labels.shape) != (B, S):
            raise ValueError(f"labels shape {tuple(labels.shape)} differs from input_ids {(B, S)}")
        tgt = labels.detach().cpu().long()
    V = cfg.vocab_size
    Sp = _round_up(int(lens.max()), 128) if kernels else int(lens.max())
    pos = torch.arange(Sp)
    real = pos[None, :] < lens[:, None]
    comp = ids.gather(1, (start[:, None] + pos[None, :]).clamp(max=S - 1)).masked_fill(~real, 0)
    if bool(((comp < 0) | (comp >= V)).any()):
        raise ValueError(f"input_ids hold token ids outside [0, {V})")
    # output slot (b, t) is predicted from compact position j = t - 1 - start[b]: scored when j and j + 1 are real
    j = torch.arange(S)[None, :] - 1 - start[:, None]
    scored = (j >= 0) & (j < lens[:, None] - 1) & (tgt != IGNORE_INDEX)
    if bool((scored & ((tgt < 0) | (tgt >= V))).any()):
        raise ValueError(f"labels must lie in [0, {V}) or be {IGNORE_INDEX}")
    rows = torch.arange(B)[:, None] * Sp + j
    gidx = torch.where(scored, rows, torch.zeros_like(rows))
    lab = torch.where(scored, tgt, torch.full_like(tgt, IGNORE_INDEX))
    return comp, Sp, gidx.reshape(-1), lab.reshape(-1)


@torch.no_grad()
def score(model, input_ids: torch.Tensor, attention_mask: torch.Tensor | None = None,
          labels: torch.Tensor | None = None, fp8_weights: bool = False) -> ScoreOutput:
    """See :meth:`LlamaForCausalLM.score`."""
    cfg, ar = model.config, model.arena
    if ar.param_sharded:
        raise ValueError("score() needs the full compute weights on this rank; the arena is parameter-sharded (FULL_SHARD)")
    w_lm = ar.w("lm_head.weight")
    kernels = cfg.head_dim == 64 and TC.usable(w_lm)
    W8.check_flag(fp8_weights)
    comp, Sp, gidx, lab = _plan(cfg, input_ids, attention_mask, labels, kernels)
    fp8 = W8.fp8_weights(model) if fp8_weights else None
    B, S = input_ids.shape
    st = score_state(model, B, Sp, S, kernels)
    pb = st.pb
    pb.ids.copy_(comp.reshape(-1))
    st.gidx.copy_(gidx)
    st.labels.copy_(lab)
    delta = _layers(model, pb, pb.ids, _prompt_attend(model, pb, B, Sp, st.cos, st.sin, kernels, fp8), fp8)
    K.rmsnorm_fwd(pb.res, ar.w("model.norm.weight"), cfg.rms_norm_eps, delta=delta, out=pb.xn, rstd=pb.rstd, x_out=pb.res)
    K.embedding_fwd(st.gidx, pb.xn, out=st.xg)        # the row that predicts each output slot, in output order
    n = B * S
    logprobs = torch.empty(n, dtype=torch.float32, device=ar.device)
    greedy = torch.empty(n, dtype=torch.bool, device=ar.device)
    for c0 in range(0, n, st.chunk):
        c1 = min(n, c0 + st.chunk)
        TC.lce_score(st.xg[c0:c1], w_lm, st.labels[c0:c1], st.pmax, st.psum, st.pidx, st.zlab)
        K.lce_score_finalize(st.pmax, st.psum, st.pidx, st.zlab, st.planes, st.labels[c0:c1], logprobs[c0:c1], greedy[c0:c1])
    return ScoreOutput(logprobs=logprobs.view(B, S), greedy=greedy.view(B, S))
