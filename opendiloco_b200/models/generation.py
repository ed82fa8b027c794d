"""KV-cached autoregressive generation for :class:`~opendiloco_b200.models.llama.LlamaForCausalLM`.

Every pass over the model is one layer program (``_layers``) on rows of this module's own (``Rows``):

    embedding -> per layer: rmsnorm -> attend -> o-proj -> rmsnorm(+residual) -> gate|up SwiGLU GEMM -> down

Only ``attend`` differs.  Prefill (and ``score``) runs the fused QKV+RoPE GEMM, copies k|v into per-layer caches and runs
the causal attention forward; the decode step runs the QKV GEMM, RoPE+append at each row's position and split-KV
attention over the cache; the verify pass of assisted generation does the same for several tokens per row.  The final
norm and the LM head (``_head``) then feed the sampler.

All the per-step scalars (positions, step counters, finished flags, sampler settings) live in device memory, so the step
is captured once into a CUDA graph and replayed (``ODB_CUDA_GRAPH=0``: eager launches); the decode step, the assisted
round and the beam step share the warm-up / capture / replay protocol (``_graphed``).  CUDA bf16 models run the
kernels of ``csrc/decode_sm90.cu`` and the training GEMMs; other precisions and devices run the same program on the
PyTorch references of :mod:`opendiloco_b200.ops`.

Assisted (speculative) generation, ``generate(assistant_model=...)``: every round the draft proposes K tokens with K
one-token decode steps (plus one more that only writes d_K into its cache), the target scores ``[last, d_1..d_K]`` in one
multi-token pass (verify attention over its cache), and one acceptance kernel keeps the longest acceptable prefix plus
one target token per row.  The whole round is one CUDA graph.  Rejected cache entries are left in place: attention reads
only up to each row's position, so moving ``pos`` back is the whole rollback.

Prompt lookup, ``generate(prompt_lookup_num_tokens=K)``: the same round without a draft model.  One kernel proposes up to K
tokens per row, the tokens that followed an earlier occurrence of the row's last n-gram in its own history (the device-side
history of the logits processors, which the acceptance kernel extends); the verify pass and a point-mass acceptance follow.

Beam search, ``generate(num_beams=...)``: transformers' deterministic beam search step for step, on B * num_beams rows of
a DecodeState of its own.  The prompts are prefilled once, into the beam-0 rows; every later step is one CUDA graph: the
decode layers, the LM head, the selection kernels and the cache reorder.  All beams of a prompt sit at the same position,
so every 128-key chunk behind the current one is immutable history: a beam that continues another row takes that row's
chunks through a per-row chunk table and copies only the current partial chunk.

FP8 weight-only mode, ``generate(fp8_weights=True)``: the layer program takes every projection weight from one helper
(``_proj``, ``_weight``, ``_mlp``).  Without FP8 weights it returns the arena weight and launches what it always did; with
them (:mod:`~opendiloco_b200.models.fp8_weights`) rows of M <= 64 run the skinny e4m3 GEMM and wider ones the bf16 GEMM on
the dequantised weights Ŵ.  Every graph key carries the mode, so switching it recaptures.

Multi-sample generation, ``generate(do_sample=True, num_return_sequences=n)``: n sibling rows per prompt (row p * n + j
is sample j of prompt p) in a DecodeState of group n.  Each prompt is prefilled once, into row p * n; its last position's
residual goes to all n rows, so the LM head and the sampler see exactly the rows of the repeated-prompt program.  A fork
then points the siblings' chunk tables at row p * n for the prompt's complete 128-key chunks and copies the partial one
into each child's own row; every decode step reads a shared chunk once for all siblings (``DK.attention_grouped``).

FP8 KV cache, ``generate(fp8_kv_cache=True)``: the DecodeState holds K and V as e4m3 with one fp32 factor per (position,
kv head) row (:mod:`~opendiloco_b200.ops.decode`); every writer quantises and every decode-time reader (the one-token step,
the verify pass, beam steps) dequantises.  The flag is part of the DecodeState and BeamState keys, so toggling it
reallocates the caches and recaptures; an assistant's own cache stays bf16.

Nothing here goes through ``LlamaEngine.workspace`` or its captured training graphs: generating between training steps
leaves the training buffers and graph untouched.
"""
from __future__ import annotations

import math
import warnings
from dataclasses import dataclass

import torch

from ..ops import attention as A
from ..ops import decode as DK
from ..ops.fp8 import E4M3
from ..ops import gemm as G
from ..ops import kernels as K
from ..ops import tc_gemm as TC
from . import fp8_weights as W8
from .llama import _use_graph

FINISHED_CHECK_EVERY = 16           # decode steps between host checks of "every row has finished"
ASSISTED_CHECK_EVERY = 4            # assisted rounds between host checks (a round emits 1 .. K+1 tokens per row)
MAX_ASSISTANT_TOKENS = 7            # verify attention: K+1 <= 8 queries per row and GQA group
DRAFT_SEED_XOR = 0x5DEECE66D        # the draft's proposals draw from a Philox stream apart from the acceptance draws


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def _resident(model, attr: str, key: tuple, make):
    """The engine's state ``attr`` if its key is ``key``, else a new one from make(); at most one is resident (the old one is
    freed before make() allocates)."""
    eng = model.engine
    st = getattr(eng, attr)
    if st is None or st.key != key:
        setattr(eng, attr, None)
        st = make()
        st.key = key
        setattr(eng, attr, st)
    return st


def _graphed(holder, key: tuple, device, run) -> None:
    """run() through holder's CUDA graph (holder.graph, holder.graph_key): the first call with a new key runs it eagerly
    (warm-up), the next one captures it and every later call replays it."""
    if holder.graph is None or holder.graph_key != key:
        if holder.graph_key != ("warm",) + key:
            holder.graph, holder.graph_key = None, ("warm",) + key
            run()
            return
        torch.cuda.synchronize(device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, capture_error_mode="thread_local"):
            run()
        holder.graph, holder.graph_key = g, key
    holder.graph.replay()


class Rows:
    """The activations of T rows of the layer program (``_layers``), one token per row: token ids, residual, normed rows,
    projection outputs, q|k|v, gate|up and SwiGLU rows.  ``att``: also the attention output (decode step, verify pass);
    prefill and scoring take theirs from the attention forward."""

    def __init__(self, cfg, T: int, device, dtype, att: bool = False):
        e = lambda *shape: torch.empty(*shape, dtype=dtype, device=device)  # noqa: E731
        h, i = cfg.hidden_size, cfg.intermediate_size
        self.T = T
        self.ids = torch.zeros(T, dtype=torch.int64, device=device)
        self.res, self.xn, self.proj = e(T, h), e(T, h), e(T, h)
        self.rstd = torch.empty(T, dtype=torch.float32, device=device)
        self.qkv, self.gu, self.act = e(T, cfg.qkv_dim), e(T, 2 * i), e(T, i)
        self.att = e(T, cfg.q_dim) if att else None


class DecodeState(Rows):
    """KV caches, the one-token rows of the decode step and device-side control scalars for B rows of up to Smax positions.
    ``fp8_kv``: the caches are e4m3 ``kv`` [L, 2, B, Hkv, Smax, D] with fp32 ``kv_inv`` [L, 2, B, Hkv, Smax] (each one
    allocation: beam search reorders all of it); ``kinv`` / ``vinv`` are the per-layer views of ``kv_inv`` (None for a bf16
    cache).  ``group`` > 1: multi-sample rows, ``group`` siblings per prompt, with the chunk table ``table`` int32 [B, Smax /
    128] of the kernel path (None otherwise, and for group 1)."""

    def __init__(self, cfg, B: int, Smax: int, device, dtype, fp8_kv: bool = False, group: int = 1):
        super().__init__(cfg, B, device, dtype, att=True)
        L, Hq, Hkv, D = cfg.num_hidden_layers, cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
        V = cfg.vocab_size
        i32 = lambda: torch.zeros(B, dtype=torch.int32, device=device)      # noqa: E731
        self.cfg, self.B, self.Smax, self.device, self.dtype = cfg, B, Smax, torch.device(device), dtype
        self.fp8_kv, self.group = fp8_kv, group
        # one allocation: beam search reorders all
        self.kv = torch.zeros(L, 2, B, Hkv, Smax, D, dtype=E4M3 if fp8_kv else dtype, device=device)
        self.kv_inv = torch.zeros(L, 2, B, Hkv, Smax, dtype=torch.float32, device=device) if fp8_kv else None
        self.kc = [self.kv[l, 0] for l in range(L)]
        self.vc = [self.kv[l, 1] for l in range(L)]
        self.kinv = [self.kv_inv[l, 0] if fp8_kv else None for l in range(L)]
        self.vinv = [self.kv_inv[l, 1] if fp8_kv else None for l in range(L)]
        n_rope = _round_up(max(cfg.max_position_embeddings, Smax), 128)
        self.cos, self.sin = K.rope_tables(n_rope, D, cfg.rope_theta, device)
        self.logits = torch.empty(B, V, dtype=dtype, device=device)
        self.pos, self.gen, self.finished, self.lens = i32(), i32(), i32(), i32()
        self.out = torch.zeros(B, Smax, dtype=torch.int64, device=device)
        self.ictl, self.fctl = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, [], device)
        # token histories of the logits processors: the real prompt tokens, then the generated ones (the sampler appends)
        self.hist = torch.zeros(B, Smax, dtype=torch.int32, device=device)
        self.proc_scratch = torch.zeros(B, 2 * ((V + 31) // 32), dtype=torch.int32, device=device)
        # sequence_bias / bad_words_ids: the fixed-capacity table and the sampler's zeroed bias rows, allocated on first use
        self.seq: DK.SeqTable | None = None
        self.seq_scratch: torch.Tensor | None = None
        self.kernels = DK.usable(self.res, D, Hq, Hkv)
        self.part_o = self.part_ml = None
        if self.kernels:
            nch = DK.attn_chunks(Smax)
            self.part_o = torch.empty(B, Hq, nch, D, dtype=torch.float32, device=device)
            self.part_ml = torch.empty(B, Hq, nch, 2, dtype=torch.float32, device=device)
        self.table = torch.zeros(B, nch, dtype=torch.int32, device=device) if self.kernels and group > 1 else None
        self.score_buf: torch.Tensor | None = None   # generate(output_scores / output_logits): see set_outputs
        self.logit_buf: torch.Tensor | None = None
        self._prefill: Rows | None = None
        self.graph = None
        self.graph_key = None

    def prefill_rows(self, T: int) -> Rows:
        """The [T = B*Sp] rows of a prefill, kept for the next prefill of the same size."""
        if self._prefill is None or self._prefill.T != T:
            self._prefill = None                      # free the old buffers before allocating the new ones
            self._prefill = Rows(self.cfg, T, self.device, self.dtype)
        return self._prefill

    def set_controls(self, do_sample: bool, temperature: float, top_k: int, top_p: float, seed: int, pad: int, eos: list[int],
                     repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0, min_new_tokens: int = 0, min_length: int = 0,
                     min_p: float = 0.0, entries: list | None = None):
        """The control blocks, and the sequence table's ``entries`` (``DK.sequence_entries``; None or empty: none).  The
        table and the sampler's bias rows are allocated the first time there are entries and rewritten in place after."""
        entries = entries or []
        if entries and self.seq is None:
            self.seq = DK.SeqTable(self.device)
            self.seq_scratch = torch.zeros(self.B, self.cfg.vocab_size, dtype=torch.float32, device=self.device)
        if self.seq is not None:
            self.seq.set(entries)
        ictl, fctl = DK.make_controls(do_sample, temperature, top_k, top_p, seed, pad, eos, "cpu", repetition_penalty,
                                      no_repeat_ngram_size, min_new_tokens, min_length, min_p, len(entries))
        self.ictl.copy_(ictl)
        self.fctl.copy_(fctl)


def set_outputs(holder, rows: int, V: int, max_new: int, scores: bool, logits: bool, pad: int, dtype) -> None:
    """generate(return_dict_in_generate=True, output_scores / output_logits): holder.score_buf fp32 and holder.logit_buf
    (the compute dtype) [max_new, rows, V], one [rows, V] row block per generated position, each allocated only when its
    flag is on (rows * max_new * V * (4 + 2) bytes with both: about 790 MB at 8 rows, 512 tokens and V = 32000) and kept
    for the next call of the same shape, so its CUDA graphs replay.  Both are filled with the padding row (-inf, 0 at
    ``pad``) here, outside any graph; the sampler, the acceptance and the beam selection overwrite the columns a live row
    emits.  A flag that is off frees its buffer."""
    for attr, on, dt in (("score_buf", scores, torch.float32), ("logit_buf", logits, dtype)):
        buf = getattr(holder, attr)
        if not on or (buf is not None and buf.shape != (max_new, rows, V)):
            setattr(holder, attr, None)
            buf = None
        if on:
            if buf is None:
                buf = torch.empty(max_new, rows, V, dtype=dt, device=holder.device)
                setattr(holder, attr, buf)
            DK.padding_rows(buf, pad)


def _out_key(holder) -> tuple:
    """The score / logit buffers a graph writes (part of every graph key, like the sequence table)."""
    return tuple(None if b is None else (b.data_ptr(), tuple(b.shape)) for b in (holder.score_buf, holder.logit_buf))


def decode_state(model, B: int, Smax: int, fp8_kv: bool = False, group: int = 1) -> DecodeState:
    """The model's decode state for (B, Smax, FP8 cache or not, siblings per prompt), allocated on first use; at most one
    is resident."""
    eng, ar = model.engine, model.arena

    def make():
        if eng.assisted_state is not None:           # its round graph reads the old caches: let them go
            eng.assisted_state.drop_graph()
        return DecodeState(model.config, B, Smax, ar.device, ar.compute_dtype, fp8_kv, group)

    return _resident(model, "decode_state", (B, Smax, str(ar.device), ar.compute_dtype, fp8_kv, group), make)


# ------------------------------------------------------------------------------------------------ layer program
def _layers(model, buf: Rows, ids: torch.Tensor, attend, fp8=None):
    """The forward layer program over the rows of ``buf``: embedding of ids, then per layer rmsnorm -> ``attend(l)`` (the
    attention output of the normed rows buf.xn: QKV GEMM, RoPE, cache writes, attention) -> o-proj -> rmsnorm(+residual)
    -> SwiGLU GEMM -> down.  Returns the last layer's output delta; the residual before it is in buf.res."""
    cfg, ar = model.config, model.arena
    eps = cfg.rms_norm_eps
    K.embedding_fwd(ids, ar.w("model.embed_tokens.weight"), out=buf.res)
    delta = None
    for l in range(cfg.num_hidden_layers):
        p = f"model.layers.{l}."
        K.rmsnorm_fwd(buf.res, ar.w(p + "input_layernorm.weight"), eps, delta=delta, out=buf.xn, rstd=buf.rstd, x_out=buf.res)
        _proj(ar, fp8, "o", l, attend(l), buf.proj)
        K.rmsnorm_fwd(buf.res, ar.w(p + "post_attention_layernorm.weight"), eps, delta=buf.proj, out=buf.xn, rstd=buf.rstd, x_out=buf.res)
        _mlp(cfg, ar, l, buf.xn, buf.gu, buf.act, fp8)
        _proj(ar, fp8, "down", l, buf.act, buf.proj)
        delta = buf.proj
    return delta


def _prompt_attend(model, buf: Rows, B: int, Sp: int, cos, sin, fused_rope: bool, fp8=None, fill=None):
    """The ``attend`` of prefill and scoring over B rows of Sp positions each, starting at position 0 (causal attention
    keeps right padding from reaching real positions): QKV(+RoPE) GEMM, ``fill(l, qkv)`` (the cache fill) on the rotated
    projections, causal attention forward."""
    cfg, ar = model.config, model.arena
    Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim

    def attend(l):
        w_qkv = _weight(ar, fp8, "qkv", l)
        if fused_rope and TC.usable(buf.xn, w_qkv):
            TC.linear_qkv_rope(buf.xn, w_qkv, buf.qkv, cos, sin, Sp, (Hq + Hkv) * D)
        else:
            _proj(ar, fp8, "qkv", l, buf.xn, buf.qkv)
            K.rope_(buf.qkv, cos, sin, Sp, Hq + Hkv, D)
        if fill is not None:
            fill(l, buf.qkv)
        return A.attention_fwd(buf.qkv, B, Sp, Hq, Hkv, D)[0]

    return attend


def _weight(ar, fp8, kind: str, l: int) -> torch.Tensor:
    """The bf16 weight of projection ``kind`` (``fp8_weights.KINDS``) of layer l: the arena's, or Ŵ in FP8 mode."""
    return W8.arena_weight(ar, kind, l) if fp8 is None else fp8.weight(kind, l)


def _proj(ar, fp8, kind: str, l: int, x, out) -> None:
    """out = x @ W^T for projection ``kind`` of layer l: the skinny FP8 GEMM where it applies, else the bf16 GEMM."""
    if fp8 is not None and fp8.skinny(kind, x):
        fp8.linear(kind, l, x, out)
    else:
        G.mm_nt(x, _weight(ar, fp8, kind, l), out=out)


def _mlp(cfg, ar, l: int, xn, gu, act, fp8=None) -> None:
    if fp8 is not None and fp8.skinny("gu", xn):
        fp8.linear("gu", l, xn, gu, act=act)
        return
    w = _weight(ar, fp8, "gu", l)
    if cfg.intermediate_size % 64 == 0 and TC.usable(xn, w):
        TC.linear_swiglu(xn, w, gu, act)
    else:
        G.mm_nt(xn, w, out=gu)
        K.swiglu_fwd(gu, out=act)


def _head(model, buf: Rows, delta, logits) -> None:
    """The final RMSNorm of buf's rows (residual + delta) and the LM-head GEMM into logits."""
    cfg, ar = model.config, model.arena
    K.rmsnorm_fwd(buf.res, ar.w("model.norm.weight"), cfg.rms_norm_eps, delta=delta, out=buf.xn, rstd=buf.rstd, x_out=buf.res)
    G.mm_nt(buf.xn, ar.w("lm_head.weight"), out=logits)


def _head_and_sample(model, st: DecodeState, delta) -> None:
    _head(model, st, delta, st.logits)
    DK.sample(st.logits, st.ictl, st.fctl, st.pos, st.gen, st.finished, st.out, st.ids, st.hist, st.proc_scratch, st.seq,
              st.seq_scratch, st.score_buf, st.logit_buf)


# ------------------------------------------------------------------------------------------------ prefill
@torch.no_grad()
def prefill(model, st: DecodeState, ids: torch.Tensor, lens: torch.Tensor, fp8=None) -> None:
    """ids [B, Sp]: prompts compacted to start at position 0 and right-padded; lens [B] real lengths; st has B * n rows,
    n = st.group.  The layers run on the B prompts once, prompt p filling cache row p * n; with n > 1 the fork makes rows
    p * n + 1 .. its children (``DK.fork``: chunk table on the kernel path, whole-row copies otherwise) and every row's
    state (pos, lens, history) is the repeated-prompt program's.  Computes the logits at position lens[p] - 1 of every row
    and samples the first token (st.pos ends at lens).  ``fp8``: the model's FP8 weights (None: the arena weights).  An
    FP8 cache (st.fp8_kv) is filled with the quantised k|v rows; the prompt's attention reads the in-flight bf16 q|k|v, so
    the first token does not depend on the cache format."""
    n, Sp = st.group, ids.shape[1]
    lr = lens.repeat_interleave(n) if n > 1 else lens
    st.lens.copy_(lr)
    st.pos.copy_(lr - 1)
    st.gen.zero_()
    st.finished.zero_()
    m = min(Sp, st.Smax)
    st.hist[:, :m].copy_(ids[:, :m].repeat_interleave(n, dim=0) if n > 1 else ids[:, :m])
    # one sample per prompt reads the lengths from st.lens, the device copy of lens
    _prefill_rows(model, st, ids, lens if n > 1 else st.lens, n, fp8)
    if n > 1:
        DK.fork(st.kv, st.table, lens, n, inv=st.kv_inv)
    _head_and_sample(model, st, st.proj)


def _prefill_rows(model, st: DecodeState, ids: torch.Tensor, lens: torch.Tensor, stride: int, fp8=None) -> None:
    """The layers over ids [B, Sp] (compacted prompts, real lengths lens [B]) once: prompt b fills cache row b * stride,
    and its last position's residual and delta rows go to decode rows b * stride .. b * stride + stride - 1 (st.res,
    st.proj), ready for the final norm and the LM head."""
    cfg = model.config
    Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    B, Sp = ids.shape
    pb = st.prefill_rows(B * Sp)
    pb.ids.copy_(ids.reshape(-1))

    def fill(l, qkv):
        DK.kv_fill(qkv, lens, st.kc[l], st.vc[l], B, Sp, Hq, Hkv, D, row_stride=stride, kinv=st.kinv[l], vinv=st.vinv[l])

    delta = _layers(model, pb, pb.ids, _prompt_attend(model, pb, B, Sp, st.cos[:Sp], st.sin[:Sp], st.kernels, fp8, fill), fp8)
    # only the last real position of every prompt feeds the LM head: gather its residual and delta rows
    last = torch.arange(B, device=st.device, dtype=torch.int64) * Sp + lens.long() - 1
    if stride > 1:
        last = last.repeat_interleave(stride)
    K.embedding_fwd(last, pb.res, out=st.res)
    K.embedding_fwd(last, delta, out=st.proj)


# ------------------------------------------------------------------------------------------------ decode step
def _one_token_layers(model, st: DecodeState, ids: torch.Tensor, table: torch.Tensor | None = None, fp8=None):
    """One token per row at st.pos: the decode layers with single-query RoPE+append and split-KV attention (through the
    chunk table, if given), on st's bf16 or FP8 cache.  Multi-sample rows (st.group > 1) attend through st's own table
    with the sibling-grouped attention."""
    cfg, ar = model.config, model.arena
    Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim

    def attend(l):
        _proj(ar, fp8, "qkv", l, st.xn, st.qkv)
        DK.rope_append(st.qkv, st.cos, st.sin, st.pos, st.kc[l], st.vc[l], Hq, Hkv, D, kinv=st.kinv[l], vinv=st.vinv[l])
        if st.group > 1:
            DK.attention_grouped(st.qkv, st.kc[l], st.vc[l], st.pos, st.att, Hq, Hkv, D, st.group, st.part_o, st.part_ml,
                                 table=st.table, kinv=st.kinv[l], vinv=st.vinv[l])
        else:
            DK.attention(st.qkv, st.kc[l], st.vc[l], st.pos, st.att, Hq, Hkv, D, st.part_o, st.part_ml, table=table,
                         kinv=st.kinv[l], vinv=st.vinv[l])
        return st.att

    return _layers(model, st, ids, attend, fp8)


def _fp8_key(fp8):
    return None if fp8 is None else fp8.token


def _step_eager(model, st: DecodeState, fp8=None) -> None:
    delta = _one_token_layers(model, st, st.ids, fp8=fp8)
    _head_and_sample(model, st, delta)


@torch.no_grad()
def step(model, st: DecodeState, graph: bool | None = None, fp8=None) -> None:
    """One decode step: consume st.ids at st.pos, sample the next token into st.ids / st.out.  With the kernels and
    ``graph`` (default: ``ODB_CUDA_GRAPH`` != 0) the first call runs eagerly (warm-up), the second captures the step and
    every call replays it.  ``fp8``: the model's FP8 weights (None: the arena weights).  Multi-sample rows (st.group > 1)
    attend through st.table; the group and the table are part of the graph key, and so is whether the state has a sequence
    table (its entries and sizes are not: the graph reads them from device memory)."""
    if graph is None:
        graph = _use_graph()
    if not (graph and st.kernels):
        _step_eager(model, st, fp8)
        return
    key = (model.arena.version, model.arena.shadow.data_ptr(), st.group, st.table.data_ptr() if st.table is not None else None,
           st.seq is not None, _out_key(st), _fp8_key(fp8))
    _graphed(st, key, st.device, lambda: _step_eager(model, st, fp8))


# ------------------------------------------------------------------------------------------------ assisted generation
class AssistedState(Rows):
    """The target's buffers of assisted generation over B rows with K proposals: the rows of the multi-token verify pass,
    (K+1)*B slot-major rows (row j*B + b is slot j of row b; ``ids`` slot 0 holds the last token, slots 1..K the
    proposals), the draft's proposal logits, the draft's own DecodeState (so a model can draft for itself, and the
    assistant's ``decode_state`` is left alone) and the round graph.  The target's caches, positions and outputs stay in
    its DecodeState.

    With ``dcfg`` None (prompt lookup) there is no draft: no draft DecodeState and no proposal logits; the proposals
    come from the target's token history, and ``cnt`` / ``proposed`` count each row's candidates."""

    def __init__(self, cfg, dcfg, B: int, K: int, Smax: int, device, dtype):
        V, D = cfg.vocab_size, cfg.head_dim
        T = (K + 1) * B
        self.B, self.K = B, K
        self.draft = DecodeState(dcfg, B, Smax, device, dtype) if dcfg is not None else None
        super().__init__(cfg, T, device, dtype, att=True)
        self.plog = torch.empty(T, V, dtype=dtype, device=device)
        self.qlog = torch.empty(K * B, V, dtype=dtype, device=device) if dcfg is not None else None
        self.stats = torch.zeros(B, 2, dtype=torch.int64, device=device)     # per row: rounds taken part in, accepted
        self.cnt = torch.zeros(B, dtype=torch.int32, device=device)          # prompt lookup: this round's candidates per row
        self.proposed = torch.zeros(B, dtype=torch.int64, device=device)     # prompt lookup: candidates proposed per row
        # the verify kernels follow the target's shapes alone; the round graph needs the draft's decode kernels too
        self.kernels = DK.usable_verify(self.res, D, cfg.num_attention_heads, cfg.num_key_value_heads)
        self.graphable = self.kernels and (self.draft is None or self.draft.kernels)
        self.part_o = self.part_ml = None
        if self.kernels:
            nsp = DK.verify_splits(Smax)
            self.part_o = torch.empty(T, cfg.num_attention_heads, nsp, D, dtype=torch.float32, device=device)
            self.part_ml = torch.empty(T, cfg.num_attention_heads, nsp, 2, dtype=torch.float32, device=device)
        self.graph = None
        self.graph_key = None
        self.graph_target = None                      # the target DecodeState the graph reads (kept alive with it)

    def drop_graph(self) -> None:
        self.graph = self.graph_key = self.graph_target = None

    def verify_passes(self) -> int:
        """Verify passes of the last generate call (rounds in which some row was still generating)."""
        return int(self.stats[:, 0].max())

    def acceptance_rate(self) -> float:
        """Accepted proposals over proposals made, over the rows and rounds of the last generate call (prompt lookup:
        over the candidates actually proposed; a row without a match proposes none)."""
        made = int(self.proposed.sum()) if self.draft is None else self.K * int(self.stats[:, 0].sum())
        return int(self.stats[:, 1].sum()) / made if made else float("nan")


def _shape(cfg) -> tuple:
    return (cfg.num_hidden_layers, cfg.hidden_size, cfg.intermediate_size, cfg.num_attention_heads, cfg.num_key_value_heads,
            cfg.head_dim, cfg.vocab_size, cfg.max_position_embeddings, cfg.rope_theta)


def assisted_state(model, assistant, B: int, K: int, Smax: int) -> AssistedState:
    """The model's assisted-generation state for (assistant shapes, B, K, Smax), allocated on first use; at most one is
    resident, on the target's engine.  ``assistant`` None: the draft-less state of prompt lookup."""
    ar = model.arena
    dcfg = assistant.config if assistant is not None else None
    key = (B, K, Smax, str(ar.device), ar.compute_dtype, _shape(dcfg) if dcfg is not None else None)
    return _resident(model, "assisted_state", key, lambda: AssistedState(model.config, dcfg, B, K, Smax, ar.device, ar.compute_dtype))


def _verify(model, tst: DecodeState, ast: AssistedState, fp8=None) -> None:
    """The target scores ast.ids (slot j at tst.pos + j) in one pass: logits of every slot -> ast.plog."""
    cfg, ar = model.config, model.arena
    Hq, Hkv, D = cfg.num_attention_heads, cfg.num_key_value_heads, cfg.head_dim
    n = ast.K + 1

    def attend(l):
        _proj(ar, fp8, "qkv", l, ast.xn, ast.qkv)
        DK.rope_append_multi(ast.qkv, tst.cos, tst.sin, tst.pos, tst.kc[l], tst.vc[l], Hq, Hkv, D, n, kinv=tst.kinv[l],
                             vinv=tst.vinv[l])
        DK.verify_attention(ast.qkv, tst.kc[l], tst.vc[l], tst.pos, ast.att, Hq, Hkv, D, n, ast.part_o, ast.part_ml,
                            kinv=tst.kinv[l], vinv=tst.vinv[l])
        return ast.att

    _head(model, ast, _layers(model, ast, ast.ids, attend, fp8), ast.plog)


def _round_eager(target, draft, tst: DecodeState, ast: AssistedState, max_new: int, ngram: int, fp8=None) -> None:
    if draft is None:                                 # prompt lookup: proposals from the history, point-mass acceptance
        DK.lookup_propose(tst.hist, tst.pos, tst.finished, tst.ictl, ast.ids, ast.cnt, ast.proposed, ngram)
        _verify(target, tst, ast, fp8)
        DK.accept(ast.plog, None, tst.ictl, tst.fctl, ast.ids, tst.pos, tst.gen, tst.finished, tst.out, max_new, None, ast.stats,
                  cnt=ast.cnt, hist=tst.hist, score_out=tst.score_buf, logit_out=tst.logit_buf)
        return
    B, Kp, dst = ast.B, ast.K, ast.draft
    for i in range(Kp + 1):
        # draft step i consumes slot i at dst.pos; steps 0..K-1 propose slot i+1, step K only writes d_K into the cache
        delta = _one_token_layers(draft, dst, ast.ids[i * B:(i + 1) * B])
        if i == Kp:
            break
        q = ast.qlog[i * B:(i + 1) * B]
        _head(draft, dst, delta, q)
        DK.sample(q, dst.ictl, dst.fctl, dst.pos, dst.gen, dst.finished, dst.out, ast.ids[(i + 1) * B:(i + 2) * B])
    _verify(target, tst, ast, fp8)                    # the draft above runs on its own weights
    DK.accept(ast.plog, ast.qlog, tst.ictl, tst.fctl, ast.ids, tst.pos, tst.gen, tst.finished, tst.out, max_new, dst.pos, ast.stats,
              score_out=tst.score_buf, logit_out=tst.logit_buf)


@torch.no_grad()
def assisted_round(target, draft, tst: DecodeState, ast: AssistedState, max_new: int, graph: bool | None = None,
                   ngram: int = 2, fp8=None) -> None:
    """One assisted round: K draft proposals, one verify pass of the target, acceptance.  ``draft`` None is a prompt-lookup
    round: up to K proposals per row from an earlier occurrence of the row's last n-gram (n <= ``ngram``) in its history,
    one verify pass, point-mass acceptance.  With the kernels and ``graph`` (default: ``ODB_CUDA_GRAPH`` != 0) the first
    call runs eagerly (warm-up), the second captures the round and every call replays it.  ``fp8``: the target's FP8
    weights (None: its arena weights); the draft always runs on its own arena weights."""
    if graph is None:
        graph = _use_graph()
    if not (graph and ast.graphable and tst.kernels):
        _round_eager(target, draft, tst, ast, max_new, ngram, fp8)
        return
    proposer = (draft.arena.version, draft.arena.shadow.data_ptr()) if draft is not None else ("lookup", ngram)
    key = (target.arena.version, target.arena.shadow.data_ptr(), *proposer, id(tst), max_new, _out_key(tst), _fp8_key(fp8))
    ast.graph_target = tst                            # id(tst) is in the key: keep tst alive while a graph may read it
    _graphed(ast, key, tst.device, lambda: _round_eager(target, draft, tst, ast, max_new, ngram, fp8))


def _check_assistant(model, assistant, P: int, max_new_tokens: int, num_assistant_tokens) -> None:
    cfg, ar = model.config, model.arena
    acfg, aar = assistant.config, assistant.arena
    if acfg.vocab_size != cfg.vocab_size:
        raise ValueError(f"assistant_model vocab_size {acfg.vocab_size} differs from the model's {cfg.vocab_size}")
    if aar.device != ar.device:
        raise ValueError(f"assistant_model is on {aar.device}, the model on {ar.device}")
    if aar.compute_dtype != ar.compute_dtype:
        raise ValueError(f"assistant_model computes in {aar.compute_dtype}, the model in {ar.compute_dtype}")
    if aar.param_sharded:
        raise ValueError("assisted generate() needs the assistant's full compute weights; its arena is parameter-sharded (FULL_SHARD)")
    if isinstance(num_assistant_tokens, bool) or not isinstance(num_assistant_tokens, int) \
            or not 1 <= num_assistant_tokens <= MAX_ASSISTANT_TOKENS:
        raise ValueError(f"num_assistant_tokens must be an integer in [1, {MAX_ASSISTANT_TOKENS}], got {num_assistant_tokens!r}")
    need = P + max_new_tokens + num_assistant_tokens
    for who, c in (("the model", cfg), ("assistant_model", acfg)):
        if need > c.max_position_embeddings:
            raise ValueError(f"prompt length {P} + max_new_tokens {max_new_tokens} + num_assistant_tokens {num_assistant_tokens} "
                             f"exceeds max_position_embeddings {c.max_position_embeddings} of {who}")


def _check_lookup(prompt_lookup_num_tokens, max_matching_ngram_size, assistant_model, num_beams, processors_on: bool, P: int,
                  max_new_tokens: int, max_position_embeddings: int) -> int:
    """Validates the prompt-lookup arguments (transformers' names); returns max_matching_ngram_size (default 2)."""
    if max_matching_ngram_size is not None and (isinstance(max_matching_ngram_size, bool) or not isinstance(max_matching_ngram_size, int)
                                                or not 1 <= max_matching_ngram_size <= DK.MAX_NGRAM):
        raise ValueError(f"max_matching_ngram_size must be an integer in [1, {DK.MAX_NGRAM}], got {max_matching_ngram_size!r}")
    ngram = 2 if max_matching_ngram_size is None else max_matching_ngram_size
    if prompt_lookup_num_tokens is None:
        return ngram
    K = prompt_lookup_num_tokens
    if isinstance(K, bool) or not isinstance(K, int) or not 1 <= K <= MAX_ASSISTANT_TOKENS:
        raise ValueError(f"prompt_lookup_num_tokens must be an integer in [1, {MAX_ASSISTANT_TOKENS}], got {K!r}")
    if assistant_model is not None:
        raise ValueError("prompt_lookup_num_tokens cannot be combined with assistant_model")
    if num_beams > 1:
        raise ValueError("prompt_lookup_num_tokens cannot be combined with num_beams > 1")
    if processors_on:
        raise ValueError("repetition_penalty, no_repeat_ngram_size and min_new_tokens are not supported yet together with "
                         "prompt_lookup_num_tokens")
    if P + max_new_tokens + K > max_position_embeddings:
        raise ValueError(f"prompt length {P} + max_new_tokens {max_new_tokens} + prompt_lookup_num_tokens {K} exceeds "
                         f"max_position_embeddings {max_position_embeddings}")
    return ngram


def _assisted_generate(model, assistant, comp, lens, P: int, max_new_tokens: int, Kp: int, controls: tuple, pad: int,
                       eos: list[int], ngram: int = 2, fp8=None, fp8_kv: bool = False, min_p: float = 0.0,
                       outputs: tuple = (False, False)) -> tuple[torch.Tensor, DecodeState]:
    """Assisted generation with ``assistant``, or prompt lookup (n-grams up to ``ngram``) with ``assistant`` None.
    Returns the new tokens and the target's DecodeState (``outputs``: its score / logit buffers, ``set_outputs``).
    ``fp8_kv``: the target's cache is FP8 (the draft's stays bf16).  ``min_p`` goes to both control blocks: the acceptance
    computes q with the target's, so the draft must draw from the same warped law."""
    B = comp.shape[0]
    Smax = _round_up(P + max_new_tokens + Kp, 128)
    tst = decode_state(model, B, Smax, fp8_kv)
    ast = assisted_state(model, assistant, B, Kp, Smax)
    dst = ast.draft
    do_sample, temperature, top_k, top_p, seed = controls
    tst.set_controls(do_sample, temperature, top_k, top_p, seed, pad, eos, min_p=min_p)
    set_outputs(tst, B, model.config.vocab_size, max_new_tokens, *outputs, pad, tst.dtype)
    if dst is not None:
        dst.set_controls(do_sample, temperature, top_k, top_p, seed ^ DRAFT_SEED_XOR, 0, [], min_p=min_p)
    tst.out.fill_(pad)
    prefill(model, tst, comp, lens, fp8)              # also leaves each row's history in tst.hist
    if dst is not None:
        prefill(assistant, dst, comp, lens)
        dst.finished.zero_()                          # the draft never stops by itself; its position follows the target's
        dst.pos.copy_(tst.pos)
    ast.ids[:B].copy_(tst.ids)
    ast.stats.zero_()
    ast.proposed.zero_()
    for r in range(max_new_tokens - 1):               # every round emits >= 1 token per unfinished row
        if r % ASSISTED_CHECK_EVERY == 0 and bool(tst.finished.all()):
            break
        assisted_round(model, assistant, tst, ast, max_new_tokens, ngram=ngram, fp8=fp8)
    return tst.out[:, :max_new_tokens].clone(), tst


# ------------------------------------------------------------------------------------------------ beam search
MAX_BEAMS = 8


@dataclass
class GenerateOutput:
    """``generate(..., return_dict_in_generate=True)``: the sequences [B * num_return_sequences, P + max_new_tokens] and,
    with beam search, the fp32 score of each (sum of its log-probabilities / generated_len ** length_penalty; None
    otherwise, multi-sample generation included).

    With ``output_scores=True`` / ``output_logits=True``: ``scores`` / ``logits``, tuples of max_new_tokens fp32 tensors
    [rows, V] (rows: the sequences' rows; beam search: B * num_beams running beams), and with beam search ``beam_indices``
    (int64 [B * num_return_sequences, max_new_tokens]: the running row that emitted each token, -1 after the hypothesis
    ends).  None when not asked for."""
    sequences: torch.Tensor
    sequences_scores: torch.Tensor | None = None
    scores: tuple[torch.Tensor, ...] | None = None
    logits: tuple[torch.Tensor, ...] | None = None
    beam_indices: torch.Tensor | None = None


class BeamState:
    """Beam search over B prompts of nb beams (row b * nb + j is beam j of prompt b): its own DecodeState for the B * nb
    rows (the model's ``decode_state`` is left alone), the selection state of ``ops.decode.beam_select``, the chunk table
    and selection partials of the kernel path, and the step graph."""

    def __init__(self, cfg, B: int, nb: int, K: int, max_new: int, Smax: int, device, dtype, fp8_kv: bool = False):
        rows = B * nb
        i32 = lambda *shape: torch.zeros(*shape, dtype=torch.int32, device=device)     # noqa: E731
        f32 = lambda *shape: torch.zeros(*shape, dtype=torch.float32, device=device)   # noqa: E731
        self.B, self.nb, self.K, self.max_new = B, nb, K, max_new
        self.dec = DecodeState(cfg, rows, Smax, device, dtype, fp8_kv)
        self.run_score, self.fin_score = f32(rows), f32(rows)
        self.fin_flag, self.parent = i32(rows), i32(rows)
        self.run_seq, self.fin_seq = i32(2, rows, max_new), i32(2, rows, max_new)
        self.unsat, self.done, self.tstep = i32(B), i32(B), i32(B)
        self.kernels = DK.usable_beam(self.dec.res, cfg.head_dim, cfg.num_attention_heads, cfg.num_key_value_heads, cfg.vocab_size,
                                      nb, Smax)
        if self.dec.kernels and not self.kernels:
            warnings.warn(f"beam search: the selection and reorder kernels take num_beams * ceil(vocab_size / 1024) <= 512 and "
                          f"at most 32768 positions (here {nb} x {DK.beam_splits(cfg.vocab_size)} and {Smax}); this run uses the "
                          "PyTorch references, with host syncs, whole-cache reorders and no CUDA graph", stacklevel=3)
        self.prompt, self.plens = i32(B, Smax), i32(B)              # the compacted prompts: the start of every beam's history
        self.table = self.part_ml = self.cand_v = self.cand_i = None
        if self.kernels:
            nsp = DK.beam_splits(cfg.vocab_size)
            self.table = i32(rows, Smax // 128)
            self.part_ml = f32(rows, nsp, 2)
            # two lists of K per split: the unpenalised and the penalised tokens (the second one only with the processors on)
            self.cand_v, self.cand_i = f32(rows, nsp, 2 * K), i32(rows, nsp, 2 * K)
        self.slot_i = self.slot_v = None             # the biased tokens of sequence_bias (kernels), with the table
        self.score_buf = self.logit_buf = None       # output_scores / output_logits (set_outputs), with the beam indices
        self.run_bi = self.fin_bi = None
        self.device = self.dec.device
        self.graph = None
        self.graph_key = None

    def reset(self, pad: int) -> None:
        """HF's initial state: running scores [0, -1e9, ...], no finished hypotheses, every table entry its own row."""
        self.run_score.view(self.B, self.nb).fill_(DK.NEG)[:, 0] = 0.0
        self.fin_score.fill_(DK.NEG)
        self.fin_flag.zero_()
        self.run_seq.fill_(pad)
        self.fin_seq.fill_(pad)
        self.unsat.fill_(1)
        self.done.zero_()
        self.tstep.zero_()
        if self.run_bi is not None:
            self.run_bi.fill_(-1)
            self.fin_bi.fill_(-1)
        if self.table is not None:
            self.table.copy_(torch.arange(self.table.shape[0], dtype=torch.int32, device=self.table.device)[:, None].expand_as(self.table))

    def set_outputs(self, scores: bool, logits: bool, pad: int) -> None:
        """The score / logit buffers of ``set_outputs`` over the running rows, and the beam indices with either."""
        rows, cfg = self.B * self.nb, self.dec.cfg
        set_outputs(self, rows, cfg.vocab_size, self.max_new, scores, logits, pad, self.dec.dtype)
        if not (scores or logits):
            self.run_bi = self.fin_bi = None
        elif self.run_bi is None:
            self.run_bi = torch.full((2, rows, self.max_new), -1, dtype=torch.int32, device=self.device)
            self.fin_bi = torch.full((2, rows, self.max_new), -1, dtype=torch.int32, device=self.device)

    def results(self, R: int) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor | None]:
        """The R best finished hypotheses of every prompt: tokens int64 [B * R, max_new], scores fp32 [B * R] and, when kept,
        their beam indices int64 [B * R, max_new] (else None)."""
        B, nb, M = self.B, self.nb, self.max_new
        par = self.tstep.long() & 1                  # each prompt's latest history buffer
        ar = torch.arange(B, device=par.device)
        seq = self.fin_seq.view(2, B, nb, M)[par, ar]
        bi = self.fin_bi.view(2, B, nb, M)[par, ar][:, :R].reshape(B * R, M).long() if self.fin_bi is not None else None
        return seq[:, :R].reshape(B * R, M).long(), self.fin_score.view(B, nb)[:, :R].reshape(B * R).clone(), bi


def beam_state(model, B: int, nb: int, K: int, max_new: int, Smax: int, fp8_kv: bool = False) -> BeamState:
    """The model's beam-search state for these shapes (and cache format), allocated on first use; at most one is resident."""
    ar = model.arena
    key = (B, nb, K, max_new, Smax, str(ar.device), ar.compute_dtype, fp8_kv)
    return _resident(model, "beam_state", key,
                     lambda: BeamState(model.config, B, nb, K, max_new, Smax, ar.device, ar.compute_dtype, fp8_kv))


@torch.no_grad()
def beam_prefill(model, bs: BeamState, ids: torch.Tensor, lens: torch.Tensor, fp8=None) -> None:
    """ids [B, Sp] compacted prompts, lens [B]: the layers run on the B prompts once and fill the beam-0 row of each
    prompt; the last position's logits go to every beam row of the prompt (st.pos ends at lens - 1)."""
    st = bs.dec
    st.pos.copy_(lens.repeat_interleave(bs.nb) - 1)
    _prefill_rows(model, st, ids, lens, bs.nb, fp8)
    _head(model, st, st.proj, st.logits)


def beam_select(bs: BeamState, length_penalty: float, early_stopping: int) -> None:
    """Select from bs.dec.logits and reorder the caches by parent."""
    st = bs.dec
    DK.beam_select(st.logits, st.ictl, bs.nb, bs.K, length_penalty, early_stopping, bs.max_new, bs.run_score, bs.fin_score,
                   bs.fin_flag, bs.run_seq, bs.fin_seq, bs.unsat, bs.done, bs.tstep, st.pos, st.ids, bs.parent, bs.part_ml,
                   bs.cand_v, bs.cand_i, fctl=st.fctl, prompt=bs.prompt, plens=bs.plens, table=st.seq, slot_i=bs.slot_i,
                   slot_v=bs.slot_v, score_out=bs.score_buf, logit_out=bs.logit_buf, run_bi=bs.run_bi, fin_bi=bs.fin_bi)
    DK.beam_reorder(st.kv, bs.table, bs.parent, st.pos, bs.nb, inv=st.kv_inv)


def _beam_step_eager(model, bs: BeamState, length_penalty: float, early_stopping: int, fp8=None) -> None:
    st = bs.dec
    delta = _one_token_layers(model, st, st.ids, bs.table, fp8)
    _head(model, st, delta, st.logits)
    beam_select(bs, length_penalty, early_stopping)


@torch.no_grad()
def beam_step(model, bs: BeamState, length_penalty: float, early_stopping: int, graph: bool | None = None, fp8=None) -> None:
    """One beam-search step: the beams' tokens at their position, the LM head, selection and reorder.  With the kernels
    and ``graph`` (default: ``ODB_CUDA_GRAPH`` != 0) the first call runs eagerly (warm-up), the second captures the step and
    every call replays it."""
    if graph is None:
        graph = _use_graph()
    if not (graph and bs.kernels):
        _beam_step_eager(model, bs, length_penalty, early_stopping, fp8)
        return
    key = (model.arena.version, model.arena.shadow.data_ptr(), float(length_penalty), int(early_stopping), bs.dec.seq is not None,
           _out_key(bs), bs.run_bi.data_ptr() if bs.run_bi is not None else None, _fp8_key(fp8))
    _graphed(bs, key, bs.dec.device, lambda: _beam_step_eager(model, bs, length_penalty, early_stopping, fp8))


def _beam_generate(model, comp, lens, Smax: int, max_new_tokens: int, nb: int, R: int, length_penalty: float, early_stopping,
                   pad: int, eos: list[int], processors: tuple = (1.0, 0, 0), fp8=None,
                   fp8_kv: bool = False, min_length: int = 0, entries: list | None = None,
                   outputs: tuple = (False, False)) -> tuple[BeamState, tuple]:
    B, Sp = comp.shape
    es = DK.EARLY_STOPPING[early_stopping]
    bs = beam_state(model, B, nb, DK.beams_to_keep(nb, len(eos)), max_new_tokens, Smax, fp8_kv)
    bs.dec.set_controls(False, 1.0, 0, 1.0, 0, pad, eos, *processors, min_length=min_length, entries=entries)
    if bs.kernels and bs.dec.seq is not None and bs.slot_i is None:
        rows = bs.B * bs.nb
        bs.slot_i = torch.zeros(rows, DK.MAX_SEQS, dtype=torch.int32, device=bs.dec.device)
        bs.slot_v = torch.zeros(rows, DK.MAX_SEQS, 2, dtype=torch.float32, device=bs.dec.device)
    bs.set_outputs(*outputs, pad)
    bs.reset(pad)
    bs.prompt[:, :Sp].copy_(comp)
    bs.plens.copy_(lens)
    beam_prefill(model, bs, comp, lens, fp8)
    beam_select(bs, length_penalty, es)              # step 0 on the prefill logits: only beam 0 has score 0
    for t in range(1, max_new_tokens):
        if t % FINISHED_CHECK_EVERY == 0 and bool(bs.done.all()):
            break
        beam_step(model, bs, length_penalty, es, fp8=fp8)
    return bs, bs.results(R)


def _check_beams(num_beams, num_return_sequences, do_sample: bool, assistant_model, early_stopping, vocab_size: int,
                 n_eos: int, prompt_lookup_num_tokens=None) -> None:
    if isinstance(num_beams, bool) or not isinstance(num_beams, int) or not 1 <= num_beams <= MAX_BEAMS:
        raise ValueError(f"num_beams must be an integer in [1, {MAX_BEAMS}], got {num_beams!r}")
    if isinstance(num_return_sequences, bool) or not isinstance(num_return_sequences, int) or num_return_sequences < 1:
        raise ValueError(f"num_return_sequences must be an integer >= 1, got {num_return_sequences!r}")
    if num_beams > 1 and num_return_sequences > num_beams:
        raise ValueError(f"num_return_sequences must be an integer in [1, num_beams={num_beams}], got {num_return_sequences!r}")
    if num_beams == 1 and num_return_sequences > 1:
        if not do_sample:
            raise ValueError(f"num_return_sequences={num_return_sequences} > 1 needs do_sample=True or num_beams >= "
                             f"num_return_sequences: greedy decoding returns one sequence per prompt")
        if assistant_model is not None or prompt_lookup_num_tokens is not None:
            raise ValueError("num_return_sequences > 1 cannot be combined with assistant_model or prompt_lookup_num_tokens")
    if not (early_stopping is True or early_stopping is False or early_stopping == "never"):
        raise ValueError(f"early_stopping must be True, False or \"never\", got {early_stopping!r}")
    if num_beams > 1 and do_sample:
        raise ValueError("beam search is deterministic here: do_sample=True cannot be combined with num_beams > 1")
    if num_beams > 1 and assistant_model is not None:
        raise ValueError("assistant_model cannot be combined with num_beams > 1")
    if num_beams > 1 and DK.beams_to_keep(num_beams, n_eos) > vocab_size:
        raise ValueError(f"num_beams {num_beams} with {n_eos} EOS ids needs a vocabulary of at least "
                         f"{DK.beams_to_keep(num_beams, n_eos)} tokens, the model has {vocab_size}")


def _check_processors(repetition_penalty, no_repeat_ngram_size, min_new_tokens, assistant_model, min_length=0, min_p=None,
                      sequence_processors: bool = False, prompt_lookup: bool = False) -> bool:
    """Validates the logits-processor arguments (HF's terms) and min_p; True when one of the processors is on.
    ``sequence_processors``: sequence_bias or bad_words_ids has entries (checked by ``DK.sequence_entries``)."""
    if isinstance(min_length, bool) or not isinstance(min_length, int) or min_length < 0:
        raise ValueError(f"min_length must be an integer >= 0 (0: off), got {min_length!r}")
    if min_p is not None and (isinstance(min_p, bool) or not isinstance(min_p, (int, float)) or not 0 <= min_p <= 1):
        raise ValueError(f"min_p must be a float in [0, 1] (None or 0: off), got {min_p!r}")
    if sequence_processors or min_length > 0:
        for on, name in ((assistant_model is not None, "assistant_model"), (prompt_lookup, "prompt_lookup_num_tokens")):
            if on:
                raise ValueError(f"sequence_bias, bad_words_ids and min_length are not supported yet together with {name}")
    if isinstance(repetition_penalty, bool) or not isinstance(repetition_penalty, (int, float)) \
            or not math.isfinite(repetition_penalty) or not repetition_penalty > 0:
        raise ValueError(f"repetition_penalty must be a finite float > 0 (1.0: off), got {repetition_penalty!r}")
    if isinstance(no_repeat_ngram_size, bool) or not isinstance(no_repeat_ngram_size, int) \
            or not 0 <= no_repeat_ngram_size <= DK.MAX_NGRAM:
        raise ValueError(f"no_repeat_ngram_size must be an integer in [0, {DK.MAX_NGRAM}] (0: off), got {no_repeat_ngram_size!r}")
    if isinstance(min_new_tokens, bool) or not isinstance(min_new_tokens, int) or min_new_tokens < 0:
        raise ValueError(f"min_new_tokens must be an integer >= 0 (0: off), got {min_new_tokens!r}")
    on = repetition_penalty != 1.0 or no_repeat_ngram_size > 0 or min_new_tokens > 0
    if on and assistant_model is not None:
        raise ValueError("repetition_penalty, no_repeat_ngram_size and min_new_tokens are not supported yet together with "
                         "assistant_model")
    return on


# ------------------------------------------------------------------------------------------------ generate
def _eos_list(eos) -> list[int]:
    if eos is None:
        return []
    if isinstance(eos, int):
        return [eos]
    return [int(e) for e in eos]


@torch.no_grad()
def generate(model, input_ids: torch.Tensor, attention_mask: torch.Tensor | None = None, max_new_tokens: int = 20,
             do_sample: bool = False, temperature: float = 1.0, top_k: int = 50, top_p: float = 1.0, eos_token_id=None,
             pad_token_id: int | None = None, seed: int = 0, assistant_model=None, num_assistant_tokens: int = 4, num_beams: int = 1,
             length_penalty: float = 1.0, early_stopping=False, num_return_sequences: int = 1,
             return_dict_in_generate: bool = False, repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0,
             min_new_tokens: int = 0, prompt_lookup_num_tokens: int | None = None,
             max_matching_ngram_size: int | None = None, fp8_weights: bool = False,
             fp8_kv_cache: bool = False, sequence_bias=None, bad_words_ids=None, min_length: int = 0,
             min_p: float | None = None, output_scores: bool = False, output_logits: bool = False) -> torch.Tensor | GenerateOutput:
    """See :meth:`LlamaForCausalLM.generate`."""
    cfg, ar = model.config, model.arena
    if ar.param_sharded:
        raise ValueError("generate() needs the full compute weights on this rank; the arena is parameter-sharded (FULL_SHARD)")
    if input_ids.dim() != 2:
        raise ValueError(f"input_ids must be [batch, prompt_length], got shape {tuple(input_ids.shape)}")
    B, P = input_ids.shape
    if max_new_tokens < 1:
        raise ValueError(f"max_new_tokens must be >= 1, got {max_new_tokens}")
    if P + max_new_tokens > cfg.max_position_embeddings:
        raise ValueError(f"prompt length {P} + max_new_tokens {max_new_tokens} exceeds max_position_embeddings "
                         f"{cfg.max_position_embeddings}")
    if do_sample and not temperature > 0:
        raise ValueError(f"temperature must be > 0 when sampling, got {temperature}")
    if do_sample and not 0 < top_p <= 1:
        raise ValueError(f"top_p must be in (0, 1], got {top_p}")
    if assistant_model is not None:
        _check_assistant(model, assistant_model, P, max_new_tokens, num_assistant_tokens)
    eos = _eos_list(cfg.eos_token_id if eos_token_id is None else eos_token_id)
    _check_beams(num_beams, num_return_sequences, do_sample, assistant_model, early_stopping, cfg.vocab_size, len(eos),
                 prompt_lookup_num_tokens)
    entries = DK.sequence_entries(sequence_bias, bad_words_ids, eos, cfg.vocab_size)
    proc_on = _check_processors(repetition_penalty, no_repeat_ngram_size, min_new_tokens, assistant_model, min_length, min_p,
                                bool(entries), prompt_lookup_num_tokens is not None)
    min_p = float(min_p or 0.0) if do_sample else 0.0          # a warper: off unless sampling, as in HF
    ngram = _check_lookup(prompt_lookup_num_tokens, max_matching_ngram_size, assistant_model, num_beams, proc_on, P, max_new_tokens,
                          cfg.max_position_embeddings)
    processors = (float(repetition_penalty), no_repeat_ngram_size, min_new_tokens)
    W8.check_flag(fp8_weights)
    if not isinstance(fp8_kv_cache, bool):
        raise ValueError(f"fp8_kv_cache must be a bool, got {fp8_kv_cache!r}")
    for name, flag in (("output_scores", output_scores), ("output_logits", output_logits)):
        if not isinstance(flag, bool):
            raise ValueError(f"{name} must be a bool, got {flag!r}")
    outputs = (output_scores and return_dict_in_generate, output_logits and return_dict_in_generate)   # as in HF
    dev = ar.device
    ids = input_ids.to(dev)
    if attention_mask is None:
        lens = torch.full((B,), P, dtype=torch.int32, device=dev)
    else:
        m = attention_mask.to(dev).bool()
        if m.shape != ids.shape:
            raise ValueError(f"attention_mask shape {tuple(m.shape)} differs from input_ids {tuple(ids.shape)}")
        if not bool((m[:, 1:] >= m[:, :-1]).all()) or not bool(m[:, -1].all()):
            raise ValueError("attention_mask must be left-padded: zeros (padding) before ones in every row")
        lens = m.sum(dim=1).to(torch.int32)
    pad = pad_token_id if pad_token_id is not None else (eos[0] if eos else 0)

    # compact each row to start at position 0, right-pad to the prefill length
    kernels = DK.usable(ar.shadow if ar.shadow is not None else ar.master, cfg.head_dim, cfg.num_attention_heads,
                        cfg.num_key_value_heads)
    max_len = int(lens.max())
    Sp = _round_up(max_len, 128) if kernels else max_len
    col = (P - lens.long())[:, None] + torch.arange(Sp, device=dev)[None, :]
    comp = ids.gather(1, col.clamp(max=P - 1))
    comp = comp.masked_fill(torch.arange(Sp, device=dev)[None, :] >= lens.long()[:, None], 0)
    fp8 = W8.fp8_weights(model) if fp8_weights else None
    if assistant_model is not None or prompt_lookup_num_tokens is not None:
        K = num_assistant_tokens if assistant_model is not None else prompt_lookup_num_tokens
        new, tst = _assisted_generate(model, assistant_model, comp, lens, P, max_new_tokens, K,
                                      (do_sample, temperature, top_k, top_p, seed), pad, eos, ngram, fp8, fp8_kv_cache, min_p, outputs)
        out = torch.cat([ids, new], dim=1)
        return GenerateOutput(out, None, *_step_outputs(tst)) if return_dict_in_generate else out
    Smax = min(_round_up(P + max_new_tokens, 128), _round_up(cfg.max_position_embeddings, 128))
    if num_beams > 1:
        bs, (new, scores, bi) = _beam_generate(model, comp, lens, Smax, max_new_tokens, num_beams, num_return_sequences, length_penalty,
                                               early_stopping, pad, eos, processors, fp8, fp8_kv_cache, min_length, entries, outputs)
        out = torch.cat([ids.repeat_interleave(num_return_sequences, dim=0), new], dim=1)
        return GenerateOutput(out, scores, *_step_outputs(bs), bi) if return_dict_in_generate else out
    n = num_return_sequences
    st = decode_state(model, B * n, Smax, fp8_kv_cache, n)

    st.set_controls(do_sample, temperature, top_k, top_p, seed, pad, eos, *processors, min_length=min_length, min_p=min_p,
                    entries=entries)
    set_outputs(st, B * n, cfg.vocab_size, max_new_tokens, *outputs, pad, st.dtype)
    st.out.fill_(pad)
    prefill(model, st, comp, lens, fp8)
    if n > 1:
        ids = ids.repeat_interleave(n, dim=0)
    for t in range(1, max_new_tokens):
        if eos and t % FINISHED_CHECK_EVERY == 0 and bool(st.finished.all()):
            break
        step(model, st, fp8=fp8)
    out = torch.cat([ids, st.out[:, :max_new_tokens].clone()], dim=1)
    return GenerateOutput(out, None, *_step_outputs(st)) if return_dict_in_generate else out


def _step_outputs(holder) -> tuple:
    """(scores, logits) of GenerateOutput from holder's buffers (``set_outputs``): copies, so the resident buffers serve the
    next call; each entry is one contiguous [rows, V] fp32 step."""
    return tuple(None if b is None else b.float().unbind(0) if b.dtype != torch.float32 else b.clone().unbind(0)
                 for b in (holder.score_buf, holder.logit_buf))
