"""Front-ends of the decode kernels (``csrc/decode_sm90.cu``) with a PyTorch reference beside each.

Dispatch follows :mod:`opendiloco_b200.ops.kernels`: tensors that qualify for the kernels (``usable``: CUDA, bf16,
head_dim 64, library symbols present) run our kernels; everything else (CPU, fp32, fp16) runs the reference, which is
also the test oracle.

KV cache layout, per layer: K and V each ``[B, Hkv, Smax, D]`` in the compute dtype.  ``pos`` (int32 ``[B]``) is the
position of each row's current token: ``rope_append`` writes at ``pos[b]`` and ``attention`` attends to keys
``0 .. pos[b]``; the sampler advances it.

Beam search keeps ``num_beams`` rows per prompt (row ``b * num_beams + j`` is beam j of prompt b) and may share cache
chunks between them: with a chunk table (int32 ``[rows, Smax / 128]``), keys ``[128 c, 128 c + 128)`` of row r live in
physical row ``table[r, c]`` (``attention``, ``beam_reorder``).

Multi-sample generation (``generate(do_sample=True, num_return_sequences=n)``) keeps n sibling rows per prompt (row
``p * n + j`` is sample j of prompt p) in the same chunk-table layout: after ``fork`` the siblings read the prompt's complete
chunks from row ``p * n``, and ``attention_grouped`` loads such a shared chunk once for all of them.

Assisted generation scores n tokens per row in one pass.  Its buffers are slot-major: row ``j*B + b`` is token j of row
b, at position ``pos[b] + j`` (``rope_append_multi``, ``verify_attention``, ``accept``).

FP8 KV cache (``generate(fp8_kv_cache=True)``): K and V are e4m3 ``[B, Hkv, Smax, D]`` with fp32 ``kinv`` / ``vinv``
``[B, Hkv, Smax]``, one power-of-two scale per (position, kv head) row by the per-row rule of :mod:`.fp8w`.  The writers
(``rope_append``, ``rope_append_multi``, ``kv_fill``) quantise the rows the bf16 writers would store (``quantize_rows_ref``
of the rotated k, and of v); the readers (``attention``, ``verify_attention``, ``gather_chunks``) see the dequantised cache
Ĉ = ``dequantize_rows(q, inv)``, and ``beam_reorder`` moves inv with the bytes.  Every function takes the inv arrays as
optional arguments: None is the bf16 cache.  Ĉ is a bf16 number for rows with amax >= 448 * 2^-125, so the kernels equal
the bf16 kernels on Ĉ bit for bit, and the references dequantise and run the bf16 references.
"""
from __future__ import annotations

import ctypes
import math

import torch

from .. import _lib
from .fp8 import E4M3
from .fp8w import dequantize_rows, quantize_rows_ref

c_void_p, c_int, c_ll, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float
_lib.register_optional("odb_dec_rope_append", [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                               c_int, c_int, c_void_p, c_void_p, c_void_p])
_lib.register_optional("odb_dec_kv_fill", [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                           c_void_p, c_void_p, c_void_p])
_lib.register_optional("odb_dec_attn_chunks", [c_int])
_lib.register_optional("odb_dec_attn", [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_int,
                                        c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p])
_lib.register_optional("odb_dec_sample", [c_void_p, c_ll, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                          c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                          c_int, c_void_p])
_lib.register_optional("odb_dec_verify_attn", [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int,
                                               c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p])
_lib.register_optional("odb_dec_accept", [c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                          c_void_p, c_void_p, c_int, c_void_p])
_lib.register_optional("odb_dec_lookup_propose", [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                                  c_int, c_int, c_void_p])
_lib.register_optional("odb_dec_beam_splits", [c_int])
_lib.register_optional("odb_dec_beam_topk", [c_void_p, c_ll, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                             c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_void_p])
_lib.register_optional("odb_dec_beam_step", [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float,
                                             c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p])
_lib.register_optional("odb_dec_beam_scores", [c_void_p, c_ll, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                               c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p])
_lib.register_optional("odb_dec_beam_reorder", [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                                c_void_p])
_lib.register_optional("odb_dec_attn_group", [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_void_p,
                                              c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_int, c_void_p])
_lib.register_optional("odb_dec_attn_group_splits", [c_int, c_int, c_int, c_int, c_int, c_int])
_lib.register_optional("odb_dec_fork", [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p])

MAX_EOS = 8
# int64 control block of the sampler: do_sample, top_k, seed, pad_token_id, n_eos, eos ids, then the logits processors'
# no_repeat_ngram_size, min_new_tokens, min_length and the number of sequence-table entries.  fp32 block: temperature,
# top_p, repetition_penalty, min_p.
CTL_DO_SAMPLE, CTL_TOP_K, CTL_SEED, CTL_PAD, CTL_N_EOS, CTL_EOS = range(6)
CTL_NGRAM = CTL_EOS + MAX_EOS
CTL_MIN_NEW = CTL_NGRAM + 1
CTL_MIN_LEN = CTL_MIN_NEW + 1
CTL_N_SEQ = CTL_MIN_LEN + 1
CTL_SIZE = CTL_N_SEQ + 1
FCTL_TEMPERATURE, FCTL_TOP_P, FCTL_PENALTY, FCTL_MIN_P = range(4)
MAX_NGRAM = 64                    # the largest no_repeat_ngram_size generate() takes (and the longest table sequence)
MAX_SAMPLE_VOCAB = 56000          # the sampler keeps one fp32 per vocabulary entry in shared memory
MAX_SEQS = 1024                   # sequence table: sequence_bias + bad_words_ids entries ...
MAX_SEQ_IDS = 16384               # ... and their ids in all
SEQ_BIAS, SEQ_BAN = 0, 1          # kinds of table entries


def usable(t: torch.Tensor, head_dim: int, Hq: int = 1, Hkv: int = 1) -> bool:
    """Our decode kernels apply: CUDA bf16, head_dim 64, a GQA group of 1, 2, 4 or 8 query heads, symbols present."""
    return (t.is_cuda and t.dtype == torch.bfloat16 and head_dim == 64 and Hq % Hkv == 0 and Hq // Hkv in (1, 2, 4, 8)
            and _lib.has_symbol("odb_dec_attn") and _lib.has_symbol("odb_dec_sample"))


def usable_verify(t: torch.Tensor, head_dim: int, Hq: int = 1, Hkv: int = 1) -> bool:
    """``usable`` plus the assisted-generation kernels (multi-token RoPE+append, verify attention, acceptance)."""
    return (usable(t, head_dim, Hq, Hkv) and _lib.has_symbol("odb_dec_verify_attn") and _lib.has_symbol("odb_dec_accept")
            and _lib.has_symbol("odb_dec_rope_append"))


def usable_beam(t: torch.Tensor, head_dim: int, Hq: int, Hkv: int, V: int, num_beams: int, Smax: int) -> bool:
    """``usable`` plus the beam-search kernels (selection over a vocabulary of V, chunk-table reorder of Smax positions)."""
    return (usable(t, head_dim, Hq, Hkv) and _lib.has_symbol("odb_dec_beam_step") and _lib.has_symbol("odb_dec_beam_reorder")
            and num_beams * beam_splits(V) <= 512 and Smax % 128 == 0 and Smax // 128 <= 256)


def beam_splits(V: int) -> int:
    """Vocabulary splits of ``beam_topk`` (1024 entries each): sizes its partials."""
    return (V + 1023) // 1024


def verify_splits(Smax: int) -> int:
    """Key tiles of 64 in a cache of Smax positions: the most splits ``verify_attention`` uses (sizes its partials)."""
    return (Smax + 63) // 64


def attn_chunks(Smax: int) -> int:
    return int(_lib.cuda_lib().odb_dec_attn_chunks(Smax))


# ------------------------------------------------------------------------------------------------ FP8 cache rows
def _ptr(t: torch.Tensor | None):
    return t.data_ptr() if t is not None else None


def _check_fp8(kc: torch.Tensor, vc: torch.Tensor, kinv: torch.Tensor | None, vinv: torch.Tensor | None) -> None:
    """The kernels' FP8 cache: e4m3 K / V with contiguous fp32 inv [B, Hkv, Smax], 16-byte aligned, Smax % 128 == 0."""
    if kinv is None:
        assert vinv is None
        return
    assert kc.dtype == E4M3 and vc.dtype == E4M3 and kinv.dtype == torch.float32 and vinv.dtype == torch.float32
    assert kinv.is_contiguous() and vinv.is_contiguous() and kinv.shape == kc.shape[:-1] and vinv.shape == vc.shape[:-1]
    assert kc.shape[2] % 128 == 0 and kinv.data_ptr() % 16 == 0 and vinv.data_ptr() % 16 == 0


def dequantize_cache(cache: torch.Tensor, inv: torch.Tensor | None, dtype: torch.dtype) -> torch.Tensor:
    """The cache as the attention reads it: Ĉ = q * inv (FP8 cache, [..., D] with inv [...]) or the cache itself."""
    if inv is None:
        return cache
    D = cache.shape[-1]
    return dequantize_rows(cache.reshape(-1, D), inv.reshape(-1), dtype).view(cache.shape)


def _store_rows(cache: torch.Tensor, inv: torch.Tensor | None, index: tuple, x: torch.Tensor) -> None:
    """cache[index] = x [..., D]; with an FP8 cache the rows of x are quantised (``quantize_rows_ref``) into the bytes of
    cache[index] and inv[index]."""
    if inv is None:
        cache[index] = x
        return
    q, iv = quantize_rows_ref(x.reshape(-1, x.shape[-1]))
    cache.view(torch.uint8)[index] = q.view(torch.uint8).view(x.shape)
    inv[index] = iv.view(x.shape[:-1])


# ------------------------------------------------------------------------------------------------ RoPE + append
def rope_append(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, pos: torch.Tensor, kc: torch.Tensor, vc: torch.Tensor,
                Hq: int, Hkv: int, D: int, kinv: torch.Tensor | None = None, vinv: torch.Tensor | None = None) -> None:
    """qkv [B, (Hq+2*Hkv)*D] (one token per row): rotate q (in place) and k at position pos[b]; k, v -> cache[b, :, pos[b]]
    (quantised with kinv / vinv: FP8 cache).  ``rope_append_multi`` with n = 1."""
    _rope_append(qkv, cos, sin, pos, kc, vc, Hq, Hkv, D, 1, kinv, vinv, usable(qkv, D, Hq, Hkv))


def kv_fill(qkv: torch.Tensor, lens: torch.Tensor, kc: torch.Tensor, vc: torch.Tensor, B: int, Sp: int, Hq: int, Hkv: int,
            D: int, row_stride: int = 1, kinv: torch.Tensor | None = None, vinv: torch.Tensor | None = None) -> None:
    """Prefill: rows s < lens[b] of the rotated packed projections qkv [B*Sp, row] -> cache[b * row_stride, :, s]
    (quantised with kinv / vinv: FP8 cache)."""
    Smax = kc.shape[2]
    if usable(qkv, D, Hq, Hkv):
        assert qkv.stride(1) == 1 and kc.is_contiguous() and vc.is_contiguous() and lens.dtype == torch.int32
        _check_fp8(kc, vc, kinv, vinv)
        _lib.check(_lib.cuda_lib().odb_dec_kv_fill(qkv.data_ptr(), qkv.stride(0), lens.data_ptr(), kc.data_ptr(), vc.data_ptr(), B, Sp,
                                                   Hq, Hkv, Smax, row_stride, _ptr(kinv), _ptr(vinv), _lib.stream_ptr(qkv)),
                   "dec_kv_fill")
        _lib.count_launch()
        return
    n = min(Sp, Smax)
    rows = qkv.view(B, Sp, -1)[:, :n]
    k = rows[..., Hq * D:(Hq + Hkv) * D].unflatten(-1, (Hkv, D)).transpose(1, 2)     # [B, Hkv, n, D]
    v = rows[..., (Hq + Hkv) * D:].unflatten(-1, (Hkv, D)).transpose(1, 2)
    keep = (torch.arange(n, device=qkv.device)[None, :] < lens.long()[:, None].to(qkv.device))[:, None, :, None]
    for cache, inv, x in ((kc, kinv, k), (vc, vinv, v)):
        if inv is None:
            d = cache[::row_stride]
            d[:, :, :n] = torch.where(keep, x, d[:, :, :n])
            continue
        q, iv = quantize_rows_ref(x.reshape(-1, D))
        d, di = cache.view(torch.uint8)[::row_stride], inv[::row_stride]
        d[:, :, :n] = torch.where(keep, q.view(torch.uint8).view(x.shape), d[:, :, :n])
        di[:, :, :n] = torch.where(keep[..., 0], iv.view(x.shape[:-1]), di[:, :, :n])


# ------------------------------------------------------------------------------------------------ decode attention
def attention(q: torch.Tensor, kc: torch.Tensor, vc: torch.Tensor, pos: torch.Tensor, out: torch.Tensor, Hq: int, Hkv: int, D: int,
              part_o: torch.Tensor | None = None, part_ml: torch.Tensor | None = None, table: torch.Tensor | None = None,
              kinv: torch.Tensor | None = None, vinv: torch.Tensor | None = None) -> torch.Tensor:
    """out[b, h*D:(h+1)*D] = softmax(q_bh . K[b, h//G, :pos[b]+1]^T / sqrt(D)) V[b, h//G, :pos[b]+1]  (one query per row).

    q: the first Hq*D columns of [B, row].  part_o fp32 [B, Hq, chunks, D] / part_ml fp32 [B, Hq, chunks, 2]: scratch of
    the split-KV kernel (``attn_chunks(Smax)`` chunks).  table: None, or the int32 chunk table [B, Smax / 128] (keys of
    chunk c of row b are read from row table[b, c]; the reference gathers them, then attends).  kinv / vinv: the FP8
    cache's inv arrays (the reference attends over Ĉ)."""
    B = q.shape[0]
    Smax = kc.shape[2]
    if usable(q, D, Hq, Hkv):
        assert q.stride(1) == 1 and out.stride(1) == 1 and kc.is_contiguous() and vc.is_contiguous() and pos.dtype == torch.int32
        _check_fp8(kc, vc, kinv, vinv)
        if table is not None:
            assert table.dtype == torch.int32 and table.is_contiguous() and table.shape == (B, attn_chunks(Smax)) and Smax % 128 == 0
        _lib.check(_lib.cuda_lib().odb_dec_attn(q.data_ptr(), q.stride(0), kc.data_ptr(), vc.data_ptr(), pos.data_ptr(), part_o.data_ptr(),
                                                part_ml.data_ptr(), out.data_ptr(), out.stride(0),
                                                table.data_ptr() if table is not None else None, B, Hq, Hkv, Smax,
                                                1.0 / math.sqrt(D), _ptr(kinv), _ptr(vinv), _lib.stream_ptr(q)), "dec_attn")
        _lib.count_launch(2)
        return out
    kc, vc = dequantize_cache(kc, kinv, q.dtype), dequantize_cache(vc, vinv, q.dtype)
    if table is not None:
        kc, vc = gather_chunks(kc, table), gather_chunks(vc, table)
    G = Hq // Hkv
    qf = q[:, : Hq * D].float().view(B, Hkv, G, D)
    att = torch.einsum("bkgd,bksd->bkgs", qf, kc.float()) / math.sqrt(D)
    valid = torch.arange(Smax, device=q.device)[None, :] <= pos.long().to(q.device)[:, None]
    att = att.masked_fill(~valid[:, None, None, :], float("-inf"))
    o = torch.einsum("bkgs,bksd->bkgd", torch.softmax(att, dim=-1), vc.float())
    out.copy_(o.reshape(B, Hq * D).to(out.dtype))
    return out


def gather_chunks(cache: torch.Tensor, table: torch.Tensor, inv: torch.Tensor | None = None,
                  dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """cache [rows, Hkv, Smax, D] read through the chunk table [rows, Smax / 128]: chunk c of row r from row table[r, c].
    With ``inv`` (FP8 cache) the dequantised cache Ĉ in ``dtype`` is read."""
    cache = dequantize_cache(cache, inv, dtype)
    rows, Hkv, Smax, D = cache.shape
    nch = table.shape[1]
    c5 = cache.view(rows, Hkv, nch, Smax // nch, D).transpose(1, 2)                   # [rows, nch, Hkv, 128, D]
    g = c5[table.long().to(cache.device), torch.arange(nch, device=cache.device)[None, :]]
    return g.transpose(1, 2).reshape(rows, Hkv, Smax, D)


# ------------------------------------------------------------------------------------------------ multi-sample generation
def attention_grouped(q: torch.Tensor, kc: torch.Tensor, vc: torch.Tensor, pos: torch.Tensor, out: torch.Tensor, Hq: int, Hkv: int,
                      D: int, group: int, part_o: torch.Tensor | None = None, part_ml: torch.Tensor | None = None,
                      table: torch.Tensor | None = None, kinv: torch.Tensor | None = None, vinv: torch.Tensor | None = None,
                      splits: int = 0) -> torch.Tensor:
    """``attention`` over rows of ``group`` siblings (rows p * group .. p * group + group - 1 belong to prompt p), through
    the chunk table: the kernel loads a chunk that siblings' table entries share once per CTA and computes every
    sibling's partial from it with ``attention``'s arithmetic, so out and the partials are bit-identical to ``attention``
    with the same table.  Siblings may sit at different positions.  ``splits``: 0 lets the launcher choose how many CTAs
    share one prompt's siblings (``attn_group_splits``; with an FP8 cache at G = 1 it runs ``attention``'s kernel through
    the table, which measured faster there); a positive value forces the grouped kernel with that split (tests).  The reference is
    ``attention``'s (the table gather; table None reads every row's own cache)."""
    rows = q.shape[0]
    Smax = kc.shape[2]
    if usable(q, D, Hq, Hkv):
        assert table is not None and table.dtype == torch.int32 and table.is_contiguous() and table.shape == (rows, attn_chunks(Smax))
        assert q.stride(1) == 1 and out.stride(1) == 1 and kc.is_contiguous() and vc.is_contiguous() and pos.dtype == torch.int32
        assert group >= 1 and rows % group == 0 and Smax % 128 == 0 and splits >= 0
        _check_fp8(kc, vc, kinv, vinv)
        _lib.check(_lib.cuda_lib().odb_dec_attn_group(q.data_ptr(), q.stride(0), kc.data_ptr(), vc.data_ptr(), pos.data_ptr(),
                                                      part_o.data_ptr(), part_ml.data_ptr(), out.data_ptr(), out.stride(0),
                                                      table.data_ptr(), rows, group, Hq, Hkv, Smax, 1.0 / math.sqrt(D), _ptr(kinv),
                                                      _ptr(vinv), splits, _lib.stream_ptr(q)), "dec_attn_group")
        _lib.count_launch(2)
        return out
    return attention(q, kc, vc, pos, out, Hq, Hkv, D, part_o, part_ml, table=table, kinv=kinv, vinv=vinv)


def attn_group_splits(rows: int, group: int, Hq: int, Hkv: int, Smax: int, fp8_kv: bool = False) -> int:
    """How many CTAs ``attention_grouped`` gives the siblings of one prompt at these shapes: enough that each CTA runs at
    most max(1, 4 / G) siblings (G = Hq / Hkv), and more, up to ``group``, while the (chunk, kv head, prompt, split) grid
    would not fill one wave of resident CTAs on the current device; 0 for an FP8 cache at G = 1, where ``attention``'s kernel
    runs through the table instead.  Needs the kernels and a device."""
    s = int(_lib.cuda_lib().odb_dec_attn_group_splits(rows, group, Hq, Hkv, Smax, int(fp8_kv)))
    if s < 0:
        raise RuntimeError(f"odb_dec_attn_group_splits failed with code {s}")
    return s


def fork(kv: torch.Tensor, table: torch.Tensor | None, lens: torch.Tensor, group: int, inv: torch.Tensor | None = None) -> None:
    """After prompt p was prefilled into row p * group (positions [0, lens[p]), lens int32 [P]), make rows p * group + 1 ..
    p * group + group - 1 its children.  kv: every layer's K and V, [L, 2, P * group, Hkv, Smax, D]; inv: with an FP8 cache
    (e4m3 kv), its fp32 inv [L, 2, P * group, Hkv, Smax].

    With a chunk table (the kernel path; int32 [P * group, Smax / 128], fully rewritten) the children take row p * group's
    entries for the complete chunks c < lens[p] // 128 and get a copy of the partial chunk [128 * (lens[p] // 128), lens[p])
    (with its inv) in their own row; every other entry names the row itself.  Without one, ``fork_reference`` copies whole
    rows."""
    if table is None:
        fork_reference(kv, group, inv)
        return
    L, two, rows, Hkv, Smax, D = kv.shape
    assert kv.is_cuda and kv.dtype == (torch.bfloat16 if inv is None else E4M3) and kv.is_contiguous() and two == 2 and D == 64
    assert inv is None or (inv.dtype == torch.float32 and inv.is_contiguous() and inv.shape == kv.shape[:-1])
    assert group >= 1 and rows % group == 0 and lens.shape == (rows // group,) and lens.dtype == torch.int32 and lens.is_contiguous()
    assert table.shape == (rows, Smax // 128) and table.dtype == torch.int32 and table.is_contiguous() and Smax % 128 == 0
    _lib.check(_lib.cuda_lib().odb_dec_fork(kv.data_ptr(), table.data_ptr(), lens.data_ptr(), rows // group, group, L, Hkv, Smax,
                                            _ptr(inv), _lib.stream_ptr(kv)), "dec_fork")
    _lib.count_launch()


def fork_reference(kv: torch.Tensor, group: int, inv: torch.Tensor | None = None) -> None:
    """Physical fork: every row of a group becomes a copy of the group's first row, in every layer's K and V (and an FP8
    cache's inv).  The chunk table of ``fork`` must read like this up to each prompt's length."""
    rows = kv.shape[2]
    parent = torch.arange(rows, dtype=torch.int32) // group * group
    beam_reorder_reference(kv, parent, inv)


# ------------------------------------------------------------------------------------------------ assisted generation
def rope_append_multi(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, pos: torch.Tensor, kc: torch.Tensor, vc: torch.Tensor,
                      Hq: int, Hkv: int, D: int, n: int, kinv: torch.Tensor | None = None, vinv: torch.Tensor | None = None) -> None:
    """qkv [n*B, row] slot-major: rotate q (in place) and k of row j*B + b at position pos[b] + j; k, v -> cache[b, :, pos[b] + j]
    (quantised with kinv / vinv: FP8 cache)."""
    _rope_append(qkv, cos, sin, pos, kc, vc, Hq, Hkv, D, n, kinv, vinv, usable_verify(qkv, D, Hq, Hkv))


def _rope_append(qkv, cos, sin, pos, kc, vc, Hq: int, Hkv: int, D: int, n: int, kinv, vinv, kernel: bool) -> None:
    """The body of both: ``rope_append_kernel`` on grid (B, n) when ``kernel``, else the reference."""
    B = qkv.shape[0] // n
    Smax = kc.shape[2]
    if kernel:
        assert qkv.stride(1) == 1 and kc.is_contiguous() and vc.is_contiguous() and pos.dtype == torch.int32
        _check_fp8(kc, vc, kinv, vinv)
        _lib.check(_lib.cuda_lib().odb_dec_rope_append(qkv.data_ptr(), qkv.stride(0), cos.data_ptr(), sin.data_ptr(), pos.data_ptr(),
                                                       kc.data_ptr(), vc.data_ptr(), B, n, Hq, Hkv, Smax, _ptr(kinv), _ptr(vinv),
                                                       _lib.stream_ptr(qkv)), "dec_rope_append")
        _lib.count_launch()
        return
    half = D // 2
    p = (pos.long().to(qkv.device)[None, :] + torch.arange(n, device=qkv.device)[:, None]).reshape(-1)     # [n*B]
    rows = torch.arange(B, device=qkv.device).repeat(n)
    c, s = cos[p][:, None, :], sin[p][:, None, :]
    x = qkv[:, : (Hq + Hkv) * D].float().view(n * B, Hq + Hkv, D)
    a, b = x[..., :half], x[..., half:]
    rot = torch.cat([a * c - b * s, b * c + a * s], dim=-1).to(qkv.dtype)
    qkv[:, : Hq * D] = rot[:, :Hq].reshape(n * B, Hq * D)
    _store_rows(kc, kinv, (rows, slice(None), p), rot[:, Hq:])
    _store_rows(vc, vinv, (rows, slice(None), p), qkv[:, (Hq + Hkv) * D:].view(n * B, Hkv, D))


def verify_attention(q: torch.Tensor, kc: torch.Tensor, vc: torch.Tensor, pos: torch.Tensor, out: torch.Tensor, Hq: int, Hkv: int,
                     D: int, n: int, part_o: torch.Tensor | None = None, part_ml: torch.Tensor | None = None,
                     kinv: torch.Tensor | None = None, vinv: torch.Tensor | None = None) -> torch.Tensor:
    """Attention of n queries per row, slot-major: query row j*B + b attends keys 0 .. pos[b] + j of row b (causal inside
    the block).  part_o fp32 [n*B, Hq, verify_splits(Smax), D] / part_ml fp32 [n*B, Hq, verify_splits(Smax), 2]: scratch
    of the split-KV kernel.  kinv / vinv: the FP8 cache's inv arrays (the reference attends over Ĉ)."""
    B = q.shape[0] // n
    Smax = kc.shape[2]
    if usable_verify(q, D, Hq, Hkv):
        assert n <= 8 and q.stride(1) == 1 and out.stride(1) == 1 and kc.is_contiguous() and vc.is_contiguous()
        assert pos.dtype == torch.int32 and part_o.shape[2] == verify_splits(Smax) and part_ml.shape[2] == verify_splits(Smax)
        _check_fp8(kc, vc, kinv, vinv)
        _lib.check(_lib.cuda_lib().odb_dec_verify_attn(q.data_ptr(), q.stride(0), kc.data_ptr(), vc.data_ptr(), pos.data_ptr(),
                                                       part_o.data_ptr(), part_ml.data_ptr(), out.data_ptr(), out.stride(0), B, n, Hq,
                                                       Hkv, Smax, 1.0 / math.sqrt(D), _ptr(kinv), _ptr(vinv), _lib.stream_ptr(q)),
                   "dec_verify_attn")
        _lib.count_launch(2)
        return out
    kc, vc = dequantize_cache(kc, kinv, q.dtype), dequantize_cache(vc, vinv, q.dtype)
    G = Hq // Hkv
    qf = q[:, : Hq * D].float().view(n, B, Hkv, G, D)
    att = torch.einsum("jbkgd,bksd->jbkgs", qf, kc.float()) / math.sqrt(D)
    last = pos.long().to(q.device)[None, :] + torch.arange(n, device=q.device)[:, None]                   # [n, B]
    valid = torch.arange(Smax, device=q.device)[None, None, :] <= last[:, :, None]
    att = att.masked_fill(~valid[:, :, None, None, :], float("-inf"))
    o = torch.einsum("jbkgs,bksd->jbkgd", torch.softmax(att, dim=-1), vc.float())
    out.copy_(o.reshape(n * B, Hq * D).to(out.dtype))
    return out


def accept(plog: torch.Tensor, qlog: torch.Tensor | None, ictl: torch.Tensor, fctl: torch.Tensor, tok: torch.Tensor, pos: torch.Tensor,
           gen: torch.Tensor, finished: torch.Tensor, out: torch.Tensor, max_new: int, draft_pos: torch.Tensor | None,
           stats: torch.Tensor, cnt: torch.Tensor | None = None, hist: torch.Tensor | None = None,
           score_out: torch.Tensor | None = None, logit_out: torch.Tensor | None = None) -> None:
    """The acceptance step of one assisted round (speculative sampling; Leviathan et al. 2023, Chen et al. 2023).

    plog [(K+1)*B, V]: the target's logits, slot-major, slot i predicting the token at pos[b] + i + 1; qlog [K*B, V]: the
    draft's logits for its proposals; tok [(K+1)*B]: slot 0 the row's last token, slots 1..K the proposals d_1..d_K.

    Greedy (ictl do_sample = 0, or top_k = 1): accept the longest prefix where d_i is the target's argmax, then emit the
    argmax at the first mismatch (or the bonus argmax after d_K).  Sampling: p and q are both distributions after the
    sampler's warpers (min_p included, with the same fctl for both); d_i is accepted with probability min(1, p(d_i) / q(d_i)); the first rejection draws from
    normalise(max(0, p - q)); K acceptances draw the bonus token from p_{K+1}.

    The emitted tokens go to out[b, gen[b]..] (a row stops after an EOS id or at max_new tokens; later tokens are never
    written), gen / pos / finished advance (a row that finishes keeps its pos), tok slot 0 becomes the next round's last
    token and draft_pos = pos.  Finished rows are left alone.  stats int64 [B, 2] += (1, accepted proposals) per row that
    took part.  CUDA draws use Philox keyed by (seed, row, gen[b], slot); the reference draws from a torch generator
    seeded by (seed, row, gen[b]), so the paths give different (equally distributed) samples for the same seed.

    Point-mass mode (prompt lookup): qlog None and cnt (int32 [B]) given.  Row b has cnt[b] <= K candidates in slots
    1..cnt[b] (later slots hold a filler that is never accepted) and q is a point mass on each.  Greedy: as above,
    stopping at cnt[b].  Sampling: d_i is accepted with probability p_i(d_i); the first rejection draws from p_i with d_i
    removed and renormalised; with no candidate left (slot cnt[b]) the token is drawn from p_{cnt[b]}.  This is the law of
    drawing from p and keeping the candidate while the draw equals it.  hist (int32 [B, S], or None): every emitted token
    is appended at hist[b, pos[b] + 1 ...] (positions < S), so hist[b, :pos[b] + 1] stays the row's history.  draft_pos
    may be None.

    ``score_out`` fp32 / ``logit_out`` [max_new, B, V], each optional: every emitted token writes, at its column of out,
    the score row (``score_rows``: greedy the raw values, sampling the warped p row it was accepted or drawn against) and
    the logits of the slot that produced it."""
    B = pos.shape[0]
    K = plog.shape[0] // B - 1
    V = plog.shape[1]
    assert qlog is not None or cnt is not None
    if plog.is_cuda and plog.dtype == torch.bfloat16 and _lib.has_symbol("odb_dec_accept"):
        assert plog.stride(1) == 1 and V <= MAX_SAMPLE_VOCAB and out.is_contiguous() and 1 <= K <= 7
        assert qlog is None or (qlog.stride(1) == 1 and qlog.shape[0] == K * B)
        assert cnt is None or (cnt.dtype == torch.int32 and cnt.is_contiguous())
        assert hist is None or (hist.dtype == torch.int32 and hist.is_contiguous() and hist.shape[0] == B)
        assert _check_outputs(score_out, logit_out, B, V) in (0, max_new)
        _lib.check(_lib.cuda_lib().odb_dec_accept(plog.data_ptr(), plog.stride(0), qlog.data_ptr() if qlog is not None else None,
                                                  qlog.stride(0) if qlog is not None else 0, V, K, ictl.data_ptr(), fctl.data_ptr(),
                                                  tok.data_ptr(), pos.data_ptr(), gen.data_ptr(), finished.data_ptr(), out.data_ptr(),
                                                  out.shape[1], max_new, draft_pos.data_ptr() if draft_pos is not None else None,
                                                  stats.data_ptr(), cnt.data_ptr() if cnt is not None else None,
                                                  hist.data_ptr() if hist is not None else None, hist.shape[1] if hist is not None else 0,
                                                  _ptr(score_out), _ptr(logit_out), B, _lib.stream_ptr(plog)), "dec_accept")
        _lib.count_launch()
        return
    c = ictl.tolist()
    fc = fctl.tolist()
    temperature, top_p = fc[FCTL_TEMPERATURE], fc[FCTL_TOP_P]
    min_p = fc[FCTL_MIN_P] if len(fc) > FCTL_MIN_P else 0.0
    greedy = not (c[CTL_DO_SAMPLE] and c[CTL_TOP_K] != 1)
    eos = set(c[CTL_EOS:CTL_EOS + c[CTL_N_EOS]])
    p_all = plog.float().view(K + 1, B, V)
    q_all = qlog.float().view(K, B, V) if qlog is not None else None
    t = tok.view(K + 1, B)
    for b in range(B):
        if finished[b]:
            if draft_pos is not None:
                draft_pos[b] = pos[b]
            continue
        g0 = int(gen[b])
        n_cand = K if cnt is None else min(max(int(cnt[b]), 0), K)
        drafts = [int(t[i + 1, b]) for i in range(n_cand)]
        n_acc, t_new = 0, 0
        if greedy:
            am = p_all[:, b].argmax(dim=-1).tolist()
            while n_acc < n_cand and drafts[n_acc] == am[n_acc]:
                n_acc += 1
            t_new = am[n_acc]
        else:
            rng = torch.Generator(device="cpu").manual_seed((int(c[CTL_SEED]) * 1000003 + b * 7919 + g0) & ((1 << 63) - 1))
            p = torch.softmax(warp_logits(p_all[:, b].cpu(), temperature, c[CTL_TOP_K], top_p, min_p), dim=-1)          # [K+1, V]
            q = (torch.softmax(warp_logits(q_all[:, b].cpu(), temperature, c[CTL_TOP_K], top_p, min_p), dim=-1)
                 if q_all is not None else None)
            while n_acc < n_cand:
                d = drafts[n_acc]
                u = float(torch.rand((), generator=rng))
                qd = q[n_acc, d] if q is not None else 1.0
                if p[n_acc, d] > 0 and u * qd <= p[n_acc, d]:
                    n_acc += 1
                    continue
                if q is not None:
                    res = (p[n_acc] - q[n_acc]).clamp(min=0)
                else:
                    res = p[n_acc].clone()
                    res[d] = 0
                t_new = int(torch.multinomial(res if float(res.sum()) > 0 else p[n_acc], 1, generator=rng))
                break
            else:
                t_new = int(torch.multinomial(p[n_cand], 1, generator=rng))
        g, fin = g0, False
        for x in drafts[:n_acc] + [t_new]:
            if fin or g >= max_new:
                break
            out[b, g] = x
            if score_out is not None:
                score_out[g, b] = score_rows(p_all[g - g0, b][None], c, fc)[0].to(score_out.device)
            if logit_out is not None:
                logit_out[g, b] = plog.view(K + 1, B, V)[g - g0, b]
            if hist is not None and int(pos[b]) + 1 + g - g0 < hist.shape[1]:
                hist[b, int(pos[b]) + 1 + g - g0] = x
            g += 1
            fin = x in eos
        fin = fin or g >= max_new
        stats[b, 0] += 1
        stats[b, 1] += n_acc
        if fin:
            finished[b] = 1
        else:
            pos[b] += n_acc + 1
        gen[b] = g
        t[0, b] = t_new
        if draft_pos is not None:
            draft_pos[b] = pos[b]


def lookup_propose(hist: torch.Tensor, pos: torch.Tensor, finished: torch.Tensor, ictl: torch.Tensor, tok: torch.Tensor,
                   cnt: torch.Tensor, proposed: torch.Tensor, ngram: int) -> None:
    """The proposals of one prompt-lookup round (transformers' ``PromptLookupCandidateGenerator``, every row at once).

    Row b's history is h = hist[b, :L] with L = pos[b] + 1 (int32 [B, S]: the real prompt tokens, then the generated
    ones).  For n from min(ngram, L - 1) down to 1: the earliest start s with h[s:s+n] == h[L-n:L] and s + n < L; the
    first n that has one wins, and its candidates are h[s+n : min(s+n+K, L)], cut before the first EOS id of ictl.  No
    such n: no candidates.  tok [(K+1)*B] slot-major: slots 1..c of row b get the c candidates, slots c+1..K the filler
    id 0; cnt[b] = c (int32) and proposed[b] += c (int64).  Finished rows are left alone.  CUDA tensors run
    ``lookup_propose_kernel``, others ``lookup_propose_reference``; both give the same result."""
    B = pos.shape[0]
    K = tok.shape[0] // B - 1
    if hist.is_cuda and _lib.has_symbol("odb_dec_lookup_propose"):
        assert hist.dtype == torch.int32 and hist.is_contiguous() and hist.shape[0] == B and pos.dtype == torch.int32
        assert cnt.dtype == torch.int32 and proposed.dtype == torch.int64 and tok.dtype == torch.int64 and 1 <= ngram <= MAX_NGRAM
        _lib.check(_lib.cuda_lib().odb_dec_lookup_propose(hist.data_ptr(), hist.shape[1], pos.data_ptr(), finished.data_ptr(),
                                                          ictl.data_ptr(), tok.data_ptr(), cnt.data_ptr(), proposed.data_ptr(), K,
                                                          ngram, B, _lib.stream_ptr(hist)), "dec_lookup_propose")
        _lib.count_launch()
        return
    lookup_propose_reference(hist, pos, finished, ictl, tok, cnt, proposed, ngram)


def lookup_candidates(h: list[int], K: int, ngram: int, eos) -> list[int]:
    """The rule of ``lookup_propose`` on one history h (a list of ids): up to K candidate ids."""
    L = len(h)
    for n in range(min(ngram, L - 1), 0, -1):
        tail = h[L - n:]
        for s in range(L - n):                                     # s + n < L
            if h[s:s + n] == tail:
                cand = h[s + n:min(s + n + K, L)]
                cut = next((i for i, x in enumerate(cand) if x in eos), len(cand))
                return cand[:cut]
    return []


def lookup_propose_reference(hist: torch.Tensor, pos: torch.Tensor, finished: torch.Tensor, ictl: torch.Tensor, tok: torch.Tensor,
                             cnt: torch.Tensor, proposed: torch.Tensor, ngram: int) -> None:
    """``lookup_propose`` in PyTorch, row by row (``lookup_candidates``)."""
    B = pos.shape[0]
    K = tok.shape[0] // B - 1
    c = ictl.tolist()
    eos = set(c[CTL_EOS:CTL_EOS + c[CTL_N_EOS]])
    t = tok.view(K + 1, B)
    for b in range(B):
        if finished[b]:
            continue
        L = min(int(pos[b]) + 1, hist.shape[1])
        cand = lookup_candidates(hist[b, :L].tolist(), K, ngram, eos)
        t[1:, b] = torch.tensor(cand + [0] * (K - len(cand)), dtype=t.dtype)
        cnt[b] = len(cand)
        proposed[b] += len(cand)


# ------------------------------------------------------------------------------------------------ beam search
EARLY_STOPPING = {False: 0, True: 1, "never": 2}    # codes of HF's early_stopping values
NEG = -1.0e9                                          # HF's score offset of a continuation that must not be chosen


def beams_to_keep(num_beams: int, n_eos: int) -> int:
    """Candidates taken per prompt and step (HF): enough that num_beams of them are not EOS."""
    return max(2, 1 + n_eos) * num_beams


def beam_select(logits: torch.Tensor, ictl: torch.Tensor, num_beams: int, K: int, length_penalty: float, early_stopping: int,
                max_new: int, run_score: torch.Tensor, fin_score: torch.Tensor, fin_flag: torch.Tensor, run_seq: torch.Tensor,
                fin_seq: torch.Tensor, unsat: torch.Tensor, done: torch.Tensor, tstep: torch.Tensor, pos: torch.Tensor,
                ids_next: torch.Tensor, parent: torch.Tensor, part_ml: torch.Tensor | None = None, cand_v: torch.Tensor | None = None,
                cand_i: torch.Tensor | None = None, fctl: torch.Tensor | None = None, prompt: torch.Tensor | None = None,
                plens: torch.Tensor | None = None, table: SeqTable | None = None, slot_i: torch.Tensor | None = None,
                slot_v: torch.Tensor | None = None, score_out: torch.Tensor | None = None, logit_out: torch.Tensor | None = None,
                run_bi: torch.Tensor | None = None, fin_bi: torch.Tensor | None = None) -> None:
    """One step of deterministic beam search (transformers' ``_beam_search`` with do_sample=False) over logits
    [B * num_beams, V] (row b * num_beams + j: beam j of prompt b).

    Log-probabilities are fp32 log_softmax of the logits; the K = ``beams_to_keep`` best continuations per prompt of
    log p + run_score (ties: the lower beam * V + token) hit the stopping criteria on an EOS id of ictl or when t + 1 ==
    max_new (t = tstep[b], tokens generated so far).  The new running beams are the num_beams best of them after -1e9 on
    those that hit; the finished hypotheses (fin_score / fin_flag / fin_seq) merge the old ones with the first num_beams
    candidates that hit, scored log p / (t + 1) ** length_penalty, with HF's -1e9 rules; then the early-stop heuristic
    (``early_stopping`` code of EARLY_STOPPING) updates unsat and done.

    Writes, for prompts not yet done: ids_next (the new beams' tokens), parent (int32, the global row each new beam
    continues), run_score, pos += 1, tstep += 1, the finished state, and the histories: int32 [2, rows, max_new]
    double-buffered by the parity of t (step t reads buffer t & 1 and writes the other).  Done prompts keep everything,
    with parent = the row itself.  With the beam_topk partials (part_ml fp32 [rows, beam_splits(V), 2], cand_v fp32 /
    cand_i int32 [rows, beam_splits(V), ck >= K]) the kernels run, otherwise ``beam_step_reference``.

    Logits processors: with ``fctl`` (the fp32 control block of ``make_controls``), ``prompt`` (int32 [B, S]: the
    compacted prompts) and ``plens`` (int32 [B]) given and the processors on in the control blocks, they apply to the
    fp32 log-probs as in HF's ``_beam_search``: log_softmax of the unprocessed row, then ``process_logits_reference``'s
    rules (not renormalised), then + run_score.  Beam row r of prompt b has the history ``prompt[b, :plens[b]]`` followed
    by ``run_seq[t & 1, r, :t]`` and has generated t tokens; at step 0 that is the prompt alone.  Scores are then sums of
    processed log-probs.  The kernel path needs ck >= 2K: beam_topk lists each split's best unpenalised and best penalised
    tokens apart, and beam_step maps both to processed scores and merges them.

    ``table``: the ``SeqTable`` of sequence_bias / bad_words_ids.  On the kernel path its biased tokens are monotone with
    neither list, so beam_topk writes each row's matched, unbanned biased tokens to slots (slot_i int32 / slot_v fp32
    [rows, MAX_SEQS] / [rows, MAX_SEQS, 2]: token, then raw logit and summed bias) and beam_step scores them exactly and
    merges them with the lists.

    generate's ``output_scores`` / ``output_logits`` (each optional, for prompts not yet done): ``score_out`` fp32 [max_new,
    rows, V] takes, at column t, every beam row's processed log-probs (HF's ``log_probs``: the values ranked before the
    running score is added; the kernel path launches ``beam_scores_kernel`` for them), ``logit_out`` [max_new, rows, V]
    the logits.  ``run_bi`` / ``fin_bi`` (int32 [2, rows, max_new], -1 where nothing was emitted) are the beam indices of
    the running and finished hypotheses, kept like run_seq / fin_seq: entry t is the global row whose token t it is."""
    proc = (fctl is not None and prompt is not None and plens is not None)
    if part_ml is None:
        beam_step_reference(logits, ictl, num_beams, K, length_penalty, early_stopping, max_new, run_score, fin_score, fin_flag, run_seq,
                            fin_seq, unsat, done, tstep, pos, ids_next, parent, fctl=fctl if proc else None, prompt=prompt, plens=plens,
                            table=table, score_out=score_out, logit_out=logit_out, run_bi=run_bi, fin_bi=fin_bi)
        return
    rows, V = logits.shape
    ck = cand_v.shape[2]
    assert logits.is_cuda and logits.dtype == torch.bfloat16 and logits.stride(1) == 1 and rows % num_beams == 0
    assert part_ml.shape == (rows, beam_splits(V), 2) and cand_v.shape == (rows, beam_splits(V), ck) and cand_i.shape == cand_v.shape
    assert ck >= (2 * K if proc else K) and cand_v.is_contiguous() and cand_i.is_contiguous()
    assert run_seq.shape == (2, rows, max_new) and fin_seq.shape == (2, rows, max_new) and run_seq.dtype == torch.int32
    if proc:
        assert prompt.dtype == torch.int32 and prompt.is_contiguous() and prompt.shape[0] == rows // num_beams
        assert plens.dtype == torch.int32 and fctl.dtype == torch.float32
    tab = proc and table is not None
    if tab:
        assert slot_i.shape == (rows, MAX_SEQS) and slot_i.dtype == torch.int32 and slot_i.is_contiguous()
        assert slot_v.shape == (rows, MAX_SEQS, 2) and slot_v.dtype == torch.float32 and slot_v.is_contiguous()
    assert _check_outputs(score_out, logit_out, rows, V) in (0, max_new)
    assert (run_bi is None) == (fin_bi is None) and (run_bi is None or (run_bi.shape == run_seq.shape and run_bi.dtype == torch.int32
                                                                         and fin_bi.shape == run_seq.shape and fin_bi.dtype == torch.int32))
    st = _lib.stream_ptr(logits)
    fp = fctl.data_ptr() if proc else None
    _lib.check(_lib.cuda_lib().odb_dec_beam_topk(logits.data_ptr(), logits.stride(0), V, K, ck, part_ml.data_ptr(), cand_v.data_ptr(),
                                                 cand_i.data_ptr(), ictl.data_ptr(), fp, prompt.data_ptr() if proc else None,
                                                 prompt.shape[1] if proc else 0, plens.data_ptr() if proc else None, run_seq.data_ptr(),
                                                 tstep.data_ptr(), num_beams, max_new, rows, table.ints.data_ptr() if tab else None,
                                                 table.bias.data_ptr() if tab else None, slot_i.data_ptr() if tab else None,
                                                 slot_v.data_ptr() if tab else None, st), "dec_beam_topk")
    if score_out is not None or logit_out is not None:
        _lib.check(_lib.cuda_lib().odb_dec_beam_scores(logits.data_ptr(), logits.stride(0), V, part_ml.data_ptr(), ictl.data_ptr(), fp,
                                                       prompt.data_ptr() if proc else None, prompt.shape[1] if proc else 0,
                                                       plens.data_ptr() if proc else None, run_seq.data_ptr(), tstep.data_ptr(),
                                                       done.data_ptr(), num_beams, max_new, rows, table.ints.data_ptr() if tab else None,
                                                       table.bias.data_ptr() if tab else None, _ptr(score_out), _ptr(logit_out), st),
                   "dec_beam_scores")
        _lib.count_launch()
    _lib.check(_lib.cuda_lib().odb_dec_beam_step(part_ml.data_ptr(), cand_v.data_ptr(), cand_i.data_ptr(), V, num_beams, K, ck,
                                                 ictl.data_ptr(), fp, float(length_penalty), int(early_stopping), max_new,
                                                 run_score.data_ptr(), fin_score.data_ptr(), fin_flag.data_ptr(), run_seq.data_ptr(),
                                                 fin_seq.data_ptr(), unsat.data_ptr(), done.data_ptr(), tstep.data_ptr(), pos.data_ptr(),
                                                 ids_next.data_ptr(), parent.data_ptr(), slot_i.data_ptr() if tab else None,
                                                 slot_v.data_ptr() if tab else None, _ptr(run_bi), _ptr(fin_bi), rows // num_beams, st),
               "dec_beam_step")
    _lib.count_launch(2)


def beam_step_reference(logits: torch.Tensor, ictl: torch.Tensor, num_beams: int, K: int, length_penalty: float, early_stopping: int,
                        max_new: int, run_score: torch.Tensor, fin_score: torch.Tensor, fin_flag: torch.Tensor, run_seq: torch.Tensor,
                        fin_seq: torch.Tensor, unsat: torch.Tensor, done: torch.Tensor, tstep: torch.Tensor, pos: torch.Tensor,
                        ids_next: torch.Tensor, parent: torch.Tensor, fctl: torch.Tensor | None = None,
                        prompt: torch.Tensor | None = None, plens: torch.Tensor | None = None, table: SeqTable | None = None,
                        score_out: torch.Tensor | None = None, logit_out: torch.Tensor | None = None,
                        run_bi: torch.Tensor | None = None, fin_bi: torch.Tensor | None = None) -> None:
    """``beam_select`` in PyTorch: transformers' ``_get_top_k_continuations``, ``_get_running_beams_for_next_iteration``,
    ``_update_finished_beams`` and ``_check_early_stop_heuristic`` over [B, num_beams, ...], with stable sorts for the
    tie rule (-inf ties included: the lower beam * V + token).  With fctl / prompt / plens, the logits processors as
    described in ``beam_select``."""
    rows, V = logits.shape
    nb = num_beams
    B = rows // nb
    dev = run_score.device
    c = ictl.tolist()
    eos = torch.tensor(c[CTL_EOS:CTL_EOS + c[CTL_N_EOS]], dtype=torch.int64, device=dev)
    t = tstep.long()
    ts = [int(x) for x in t.tolist()]
    live = done == 0
    top = lambda x, k: torch.sort(x, dim=1, descending=True, stable=True).indices[:, :k]   # noqa: E731
    # c. top-K continuations
    logp = torch.log_softmax(logits.float(), dim=-1).to(dev)
    fc = fctl.tolist() if fctl is not None else []
    if prompt is not None and plens is not None and processors_on(c, fc):
        tr = t.to(dev).repeat_interleave(nb)
        logp = process_logits_reference(logp, beam_histories(prompt, plens, run_seq, tstep, nb), plens.long().to(dev).repeat_interleave(nb) + tr,
                                        tr, fc[FCTL_PENALTY], c[CTL_NGRAM], c[CTL_MIN_NEW], c[CTL_EOS:CTL_EOS + c[CTL_N_EOS]],
                                        _table_entries(table, c), c[CTL_MIN_LEN])
    lr = live.repeat_interleave(nb)
    col = t.to(dev).repeat_interleave(nb)[lr]
    if score_out is not None:
        score_out[col, lr.nonzero()[:, 0]] = logp[lr]
    if logit_out is not None:
        logit_out[col, lr.nonzero()[:, 0]] = logits.to(dev)[lr]
    logp = logp.view(B, nb, V) + run_score.view(B, nb, 1)
    idx = top(logp.view(B, nb * V), K)
    vals = logp.view(B, nb * V).gather(1, idx)
    beam, tok = idx // V, idx % V
    # d. stopping criteria
    last = (t + 1 >= max_new)[:, None]
    hits = last | torch.isin(tok, eos)
    # e. running beams of the next step
    trs = vals + hits.float() * NEG
    rsel = top(trs, nb)
    new_rs = trs.gather(1, rsel)
    # f. finished hypotheses
    just = hits & (torch.arange(K, device=dev) < nb)[None, :]
    denom = torch.tensor([float((x + 1) ** float(length_penalty)) for x in ts], dtype=torch.float32, device=dev)
    f = vals / denom[:, None]
    fs_old, ff_old = fin_score.view(B, nb), fin_flag.view(B, nb) != 0
    f = f + (ff_old.all(1, keepdim=True) & (early_stopping == 1)).float() * NEG
    f = f + (unsat.view(B, 1) == 0).float() * NEG
    f = f + (~just).float() * NEG
    merged = torch.cat([fs_old, f], dim=1)
    msel = top(merged, nb)
    new_fs = merged.gather(1, msel)
    new_ff = torch.cat([ff_old, just], dim=1).gather(1, msel)
    # histories: candidate k = the running history of its beam + its token at t
    M = max_new
    ar = torch.arange(B, device=dev)
    par = t & 1
    run_all, fin_all = run_seq.view(2, B, nb, M), fin_seq.view(2, B, nb, M)
    cand = run_all[par, ar].gather(1, beam[:, :, None].expand(B, K, M))
    cand = torch.where(torch.arange(M, device=dev)[None, None, :] == t[:, None, None], tok[:, :, None].to(cand.dtype), cand)
    new_run = cand.gather(1, rsel[:, :, None].expand(B, nb, M))
    new_fin = torch.cat([fin_all[par, ar], cand], dim=1).gather(1, msel[:, :, None].expand(B, nb, M))
    if run_bi is not None:                       # the same gathers, with the candidate's global parent row at t
        rbi, fbi = run_bi.view(2, B, nb, M), fin_bi.view(2, B, nb, M)
        cbi = rbi[par, ar].gather(1, beam[:, :, None].expand(B, K, M))
        cbi = torch.where(torch.arange(M, device=dev)[None, None, :] == t[:, None, None], (ar[:, None] * nb + beam)[:, :, None].to(cbi.dtype),
                          cbi)
        new_rbi = cbi.gather(1, rsel[:, :, None].expand(B, nb, M))
        new_fbi = torch.cat([fbi[par, ar], cbi], dim=1).gather(1, msel[:, :, None].expand(B, nb, M))
    # g. early-stop heuristic
    best_len = [max_new if (early_stopping == 2 and length_penalty > 0) else x + 1 for x in ts]
    bden = torch.tensor([float(n ** float(length_penalty)) for n in best_len], dtype=torch.float32, device=dev)
    best_possible = new_rs[:, :1] / bden[:, None]
    worst = torch.where(new_ff, new_fs.min(dim=1, keepdim=True).values, torch.full_like(new_fs, NEG))
    new_unsat = (unsat != 0) & (best_possible > worst).any(dim=1)
    new_done = ~new_unsat | ((early_stopping == 1) & new_ff.all(dim=1)) | last[:, 0]
    # write back the prompts that were not done
    run_all[1 - par[live], ar[live]] = new_run[live]
    fin_all[1 - par[live], ar[live]] = new_fin[live]
    if run_bi is not None:
        rbi[1 - par[live], ar[live]] = new_rbi[live]
        fbi[1 - par[live], ar[live]] = new_fbi[live]
    run_score.copy_(torch.where(lr, new_rs.reshape(-1), run_score))
    fin_score.copy_(torch.where(lr, new_fs.reshape(-1), fin_score))
    fin_flag.copy_(torch.where(lr, new_ff.reshape(-1).to(fin_flag.dtype), fin_flag))
    rows_idx = torch.arange(rows, device=dev)
    parent.copy_(torch.where(lr, (ar[:, None] * nb + beam.gather(1, rsel)).reshape(-1), rows_idx).to(parent.dtype))
    ids_next.copy_(torch.where(lr, tok.gather(1, rsel).reshape(-1), ids_next))
    pos.add_(lr.to(pos.dtype))
    unsat.copy_(torch.where(live, new_unsat.to(unsat.dtype), unsat))
    done.copy_(torch.where(live, new_done.to(done.dtype), done))
    tstep.add_(live.to(tstep.dtype))


def beam_histories(prompt: torch.Tensor, plens: torch.Tensor, run_seq: torch.Tensor, tstep: torch.Tensor, num_beams: int) -> torch.Tensor:
    """Every beam row's history, compacted: [rows, S + max_new] int64 whose row r (prompt b = r // num_beams) holds
    prompt[b, :plens[b]], then run_seq[t & 1, r, :t] with t = tstep[b]; the rest is -1."""
    dev = run_seq.device
    _, rows, M = run_seq.shape
    S = prompt.shape[1]
    lens = plens.long().to(dev).repeat_interleave(num_beams)
    t = tstep.long().to(dev).repeat_interleave(num_beams)
    col = torch.arange(S + M, device=dev)[None, :]
    r = torch.arange(rows, device=dev)
    run = run_seq[t & 1, r].long()                                                     # [rows, M]
    pr = prompt.to(dev).long().repeat_interleave(num_beams, dim=0)
    from_prompt = pr.gather(1, col.clamp(max=S - 1).expand(rows, -1))
    from_run = run.gather(1, (col - lens[:, None]).clamp(0, M - 1))
    h = torch.where(col < lens[:, None], from_prompt, from_run)
    return torch.where(col < (lens + t)[:, None], h, torch.full_like(h, -1))


def beam_reorder(kv: torch.Tensor, table: torch.Tensor | None, parent: torch.Tensor, pos: torch.Tensor, num_beams: int,
                 inv: torch.Tensor | None = None) -> None:
    """After a selection, make every beam row's cache the history of its parent row (int32 [rows], pos: the next position
    to write, the same for all beams of a prompt).  kv: every layer's K and V of the beam rows, [L, 2, rows, Hkv, Smax, D];
    inv: with an FP8 cache (e4m3 kv), its fp32 inv [L, 2, rows, Hkv, Smax], moved with the bytes.

    With a chunk table (the kernel path), complete 128-position chunks are shared: a child whose parent is another row
    takes the parent's table entries below pos // 128 and gets a copy of positions [128 * (pos // 128), pos) in its own
    row.  Without one, ``beam_reorder_reference`` moves whole rows."""
    if table is None:
        beam_reorder_reference(kv, parent, inv)
        return
    L, two, rows, Hkv, Smax, D = kv.shape
    assert kv.is_cuda and kv.dtype == (torch.bfloat16 if inv is None else E4M3) and kv.is_contiguous() and two == 2 and D == 64
    assert rows % num_beams == 0 and (inv is None or (inv.dtype == torch.float32 and inv.is_contiguous() and inv.shape == kv.shape[:-1]))
    assert table.shape == (rows, Smax // 128) and table.dtype == torch.int32 and parent.dtype == torch.int32 and pos.dtype == torch.int32
    _lib.check(_lib.cuda_lib().odb_dec_beam_reorder(kv.data_ptr(), table.data_ptr(), parent.data_ptr(), pos.data_ptr(), rows // num_beams,
                                                    num_beams, L, Hkv, Smax, _ptr(inv), _lib.stream_ptr(kv)), "dec_beam_reorder")
    _lib.count_launch()


def beam_reorder_reference(kv: torch.Tensor, parent: torch.Tensor, inv: torch.Tensor | None = None) -> None:
    """Physical reorder: row r of every layer's K and V (and of an FP8 cache's inv) becomes (a copy of) row parent[r].  The
    chunk table of ``beam_reorder`` must read exactly like this."""
    idx = parent.long().to(kv.device)
    raw = kv.view(torch.uint8) if kv.dtype == E4M3 else kv
    raw.copy_(raw.index_select(2, idx))
    if inv is not None:
        inv.copy_(inv.index_select(2, idx))


# ------------------------------------------------------------------------------------------------ sampler
def make_controls(do_sample: bool, temperature: float, top_k: int, top_p: float, seed: int, pad: int, eos: list[int], device,
                  repetition_penalty: float = 1.0, no_repeat_ngram_size: int = 0, min_new_tokens: int = 0, min_length: int = 0,
                  min_p: float = 0.0, n_seq: int = 0):
    """(ictl int64 [CTL_SIZE], fctl fp32 [4]) for ``sample``, ``accept`` and ``beam_select``.  The logits processors are
    off at their defaults (penalty 1.0, n-gram size 0, min_new_tokens 0, min_length 0, no sequence-table entries: n_seq
    counts the entries of the state's ``SeqTable``), and so is min_p (0)."""
    if len(eos) > MAX_EOS:
        raise ValueError(f"at most {MAX_EOS} EOS ids are supported, got {len(eos)}")
    ictl = [int(do_sample), int(top_k), int(seed) & ((1 << 63) - 1), int(pad), len(eos)] + list(eos) + [0] * (MAX_EOS - len(eos))
    ictl += [int(no_repeat_ngram_size), int(min_new_tokens), int(min_length), int(n_seq)]
    return (torch.tensor(ictl, dtype=torch.int64, device=device),
            torch.tensor([float(temperature), float(top_p), float(repetition_penalty), float(min_p)], dtype=torch.float32,
                         device=device))


def processors_on(ictl: list[int], fctl: list[float]) -> bool:
    """The control blocks (as lists) turn a logits processor on (the kernels' test, on the same fields)."""
    return (len(fctl) > FCTL_PENALTY and len(ictl) > CTL_N_SEQ
            and (fctl[FCTL_PENALTY] != 1.0 or ictl[CTL_NGRAM] > 0 or ictl[CTL_N_SEQ] > 0
                 or ((ictl[CTL_MIN_NEW] > 0 or ictl[CTL_MIN_LEN] > 0) and ictl[CTL_N_EOS] > 0)))


def _check_sequence(seq, vocab_size: int, what: str) -> tuple[int, ...]:
    if not isinstance(seq, (list, tuple)) or not seq:
        raise ValueError(f"{what}: every sequence must be a non-empty list of token ids, got {seq!r}")
    if len(seq) > MAX_NGRAM:
        raise ValueError(f"{what}: sequences of at most {MAX_NGRAM} ids are supported, got one of {len(seq)}")
    for t in seq:
        if isinstance(t, bool) or not isinstance(t, int) or not 0 <= t < vocab_size:
            raise ValueError(f"{what}: token ids must be integers in [0, {vocab_size}), got {t!r} in {seq!r}")
    return tuple(int(t) for t in seq)


def sequence_entries(sequence_bias, bad_words_ids, eos: list[int], vocab_size: int) -> list[tuple[tuple[int, ...], float, int]]:
    """The entries (ids, bias, kind) of a ``SeqTable`` for generate()'s ``sequence_bias`` (HF's dict ``{tuple(ids): bias}``
    or list ``[[ids], bias]`` form; later duplicates of the list form win, as HF's conversion to a dict) and
    ``bad_words_ids`` (a list of id lists; single-token entries equal to an EOS id are dropped, as HF drops them).  The
    bias entries come first, in HF's summation order: the length-1 sequences, then the longer ones, each in dict order.
    Raises ValueError for ids outside [0, vocab_size), empty or over-long (> MAX_NGRAM) sequences, a NaN or +inf bias, and
    more than MAX_SEQS entries or MAX_SEQ_IDS ids in all."""
    entries = []
    if sequence_bias is not None:
        if isinstance(sequence_bias, dict):
            items = list(sequence_bias.items())
        elif isinstance(sequence_bias, (list, tuple)):
            for it in sequence_bias:
                if not (isinstance(it, (list, tuple)) and len(it) == 2 and isinstance(it[0], (list, tuple))):
                    raise ValueError(f"sequence_bias: the list form is [[ids], bias] per entry, got {it!r}")
            items = list({tuple(it[0]): it[1] for it in sequence_bias}.items())
        else:
            raise ValueError(f"sequence_bias must be a dict {{tuple(ids): bias}} or a list of [[ids], bias], got {sequence_bias!r}")
        seqs = []
        for ids, b in items:
            ids = _check_sequence(list(ids) if isinstance(ids, tuple) else ids, vocab_size, "sequence_bias")
            if isinstance(b, bool) or not isinstance(b, (int, float)) or math.isnan(b) or b == math.inf:
                raise ValueError(f"sequence_bias: a bias must be a float that is not NaN or +inf (-inf bans), got {b!r}")
            seqs.append((ids, float(b)))
        entries += [(i, b, SEQ_BIAS) for i, b in seqs if len(i) == 1] + [(i, b, SEQ_BIAS) for i, b in seqs if len(i) > 1]
    if bad_words_ids is not None:
        if not isinstance(bad_words_ids, (list, tuple)):
            raise ValueError(f"bad_words_ids must be a list of lists of token ids, got {bad_words_ids!r}")
        for w in bad_words_ids:
            ids = _check_sequence(w, vocab_size, "bad_words_ids")
            if len(ids) == 1 and ids[0] in eos:
                continue
            entries.append((ids, -math.inf, SEQ_BAN))
    if len(entries) > MAX_SEQS or sum(len(e[0]) for e in entries) > MAX_SEQ_IDS:
        raise ValueError(f"sequence_bias and bad_words_ids take at most {MAX_SEQS} sequences and {MAX_SEQ_IDS} ids together, "
                         f"got {len(entries)} and {sum(len(e[0]) for e in entries)}")
    return entries


class SeqTable:
    """The fixed-capacity device table of ``sequence_entries``: int32 ``ints`` = offsets [MAX_SEQS + 1] | kinds [MAX_SEQS]
    | ids [MAX_SEQ_IDS] (entry e is ids[off[e], off[e + 1])) and fp32 ``bias`` [MAX_SEQS]; ``entries`` keeps the host
    copy the references read.  ``set`` rewrites it in place, so graphs that read it replay with any entries; the number in
    use is the control block's CTL_N_SEQ."""

    def __init__(self, device):
        self.ints = torch.zeros(2 * MAX_SEQS + 1 + MAX_SEQ_IDS, dtype=torch.int32, device=device)
        self.bias = torch.zeros(MAX_SEQS, dtype=torch.float32, device=device)
        self.entries: list = []

    def set(self, entries: list) -> None:
        if entries == self.entries:
            return
        assert len(entries) <= MAX_SEQS and sum(len(e[0]) for e in entries) <= MAX_SEQ_IDS
        ints = torch.zeros(self.ints.shape, dtype=torch.int32)
        off = [0]
        for ids, _, _ in entries:
            off.append(off[-1] + len(ids))
        ints[:len(off)] = torch.tensor(off, dtype=torch.int32)
        ints[MAX_SEQS + 1:MAX_SEQS + 1 + len(entries)] = torch.tensor([k for _, _, k in entries], dtype=torch.int32)
        ints[2 * MAX_SEQS + 1:2 * MAX_SEQS + 1 + off[-1]] = torch.tensor([t for ids, _, _ in entries for t in ids], dtype=torch.int32)
        bias = torch.zeros(MAX_SEQS, dtype=torch.float32)
        bias[:len(entries)] = torch.tensor([b for _, b, _ in entries], dtype=torch.float32)
        self.ints.copy_(ints)
        self.bias.copy_(bias)
        self.entries = list(entries)


def _table_entries(table: SeqTable | None, ictl: list[int]) -> list:
    return table.entries[:ictl[CTL_N_SEQ]] if table is not None and len(ictl) > CTL_N_SEQ else []


def _seq_matches(h: torch.Tensor, L: torch.Tensor, ids: tuple[int, ...]) -> torch.Tensor:
    """[rows] bool: the histories h[r, :L[r]] end with ids[:-1] and L >= len(ids) (always true for one id)."""
    k = len(ids)
    if k == 1:
        return torch.ones(h.shape[0], dtype=torch.bool, device=h.device)
    q = (L[:, None] - k + 1 + torch.arange(k - 1, device=h.device)[None, :]).clamp(0, h.shape[1] - 1)
    return (L >= k) & (h.gather(1, q) == torch.tensor(ids[:-1], dtype=h.dtype, device=h.device)[None, :]).all(dim=1)


def process_logits_reference(x: torch.Tensor, histories: torch.Tensor, lens: torch.Tensor, n_generated: torch.Tensor, penalty: float,
                             n: int, min_new: int, eos: list[int], seqs: list = (), min_len: int = 0) -> torch.Tensor:
    """HF's logits processors, in HF's order, on fp32 values x [rows, V]; returns a new tensor.  Row r's history is
    histories[r, :lens[r]] (int, [rows, S]); n_generated[r] counts the tokens it has generated.

    - Sequence bias (the SEQ_BIAS entries of ``seqs``, ``sequence_entries``): a length-1 sequence adds its bias to its
      token; a longer one adds it to its last token when the history (of length L >= its length) ends with its other
      tokens.  The biases of a token are summed from 0 in table order, then added to x once.
    - Repetition penalty (``penalty`` != 1): every distinct token of the history gets ``x < 0 ? x * p : x / p``, once.
    - N-gram ban (``n`` > 0): with h the history and L its length, if L + 1 >= n, every start s <= L - n with
      ``h[s .. s+n-2] == h[L-n+1 .. L-1]`` bans ``h[s+n-1]`` (-inf); matches may overlap, and n = 1 bans the whole history.
    - Bad words (the SEQ_BAN entries of ``seqs``): the last token of a sequence that matches as above gets -inf.
    - Min length: while L < ``min_len``, every id of ``eos`` gets -inf.
    - Min new tokens: while n_generated < ``min_new``, every id of ``eos`` gets -inf.

    HF passes the padded ``input_ids``, so for left-padded prompts it also counts the padding ids; here a history holds only
    the real prompt tokens and the generated ones."""
    rows, V = x.shape
    dev = x.device
    h = histories.to(dev).long()
    S = h.shape[1]
    L = lens.to(dev).long()
    col = torch.arange(S, device=dev)[None, :]
    x = x.clone()
    if any(k == SEQ_BIAS for _, _, k in seqs):
        bias = torch.zeros(rows, V, dtype=torch.float32, device=dev)
        for ids, b, k in seqs:
            if k == SEQ_BIAS:
                bias[:, ids[-1]] += torch.where(_seq_matches(h, L, ids), torch.tensor(b, device=dev), torch.tensor(0.0, device=dev))
        x = x + bias
    if penalty != 1.0:
        tok = torch.where((col < L[:, None]) & (h >= 0) & (h < V), h, torch.full_like(h, V))
        seen = torch.zeros(rows, V + 1, dtype=torch.bool, device=dev).scatter_(1, tok, True)[:, :V]
        x = torch.where(seen, torch.where(x < 0, x * penalty, x / penalty), x)
    ban = torch.zeros(rows, V + 1, dtype=torch.bool, device=dev)
    if n > 0 and S >= n:
        win = h.unfold(1, n, 1)                                                         # [rows, S - n + 1, n]
        q = (L[:, None] - n + 1 + torch.arange(n - 1, device=dev)[None, :]).clamp(0, S - 1)
        prefix = h.gather(1, q)                                                         # h[L-n+1 .. L-1]
        starts = torch.arange(S - n + 1, device=dev)[None, :]
        match = (win[:, :, :n - 1] == prefix[:, None, :]).all(dim=-1) & (starts <= (L - n)[:, None])
        follower = win[:, :, n - 1]
        follower = torch.where(match & (follower >= 0) & (follower < V), follower, torch.full_like(follower, V))
        ban.scatter_(1, follower, True)
    for ids, _, k in seqs:
        if k == SEQ_BAN:
            ban[:, ids[-1]] |= _seq_matches(h, L, ids)
    if eos and (min_new > 0 or min_len > 0):
        early = (n_generated.to(dev).long() < min_new) | (L < min_len)
        ban[:, torch.tensor(eos, dtype=torch.long, device=dev)] |= early[:, None]
    return x.masked_fill(ban[:, :V], float("-inf"))


def sample(logits: torch.Tensor, ictl: torch.Tensor, fctl: torch.Tensor, pos: torch.Tensor, gen: torch.Tensor, finished: torch.Tensor,
           out: torch.Tensor, ids_next: torch.Tensor, hist: torch.Tensor | None = None, scratch: torch.Tensor | None = None,
           table: SeqTable | None = None, seq_scratch: torch.Tensor | None = None, score_out: torch.Tensor | None = None,
           logit_out: torch.Tensor | None = None) -> None:
    """Pick one token per row of logits [B, V] and write it to out[b, gen[b]] and ids_next[b]; then gen += 1, pos += 1.

    Greedy (ictl do_sample = 0, or top_k = 1): argmax, ties to the lowest index.  Sampling: logits / temperature, keep the
    top_k largest (0 = all; ties with the k-th value are kept), keep the smallest set of largest probabilities whose mass
    reaches top_p (every token tied with the smallest kept one is kept too), keep the tokens whose probability is at least
    min_p times the largest (fctl min_p > 0), draw from the rest.  A row that has produced an EOS id emits ``pad`` from then
    on (``finished``).
    CUDA draws use Philox keyed by (seed, row, gen[b]); the reference draws from a torch generator seeded by (seed, step),
    so the two paths give different (equally distributed) samples for the same seed.

    hist (int32 [B, S]): the rows' token histories, row b's tokens at positions 0 .. pos[b] (the real prompt tokens, then
    the generated ones); the emitted token is appended at hist[b, pos[b] + 1] (when that is < S).  With a history and the
    processors on in the control blocks (``make_controls``), the logits first go through ``process_logits_reference``'s
    rules in fp32 (history length pos[b] + 1, gen[b] tokens generated), and greedy and sampling work on the processed
    values, which are never rounded back to bf16.  A row whose processed values are all -inf emits token 0 greedily; a
    sampled row with no finite value emits its processed argmax.  The kernel keeps two bitmaps per row in scratch (int32
    [B, 2 * ceil(V / 32)]).  ``table``: the ``SeqTable`` of sequence_bias / bad_words_ids (its first ictl CTL_N_SEQ
    entries apply); the kernel then needs ``seq_scratch``, fp32 [B, V] of zeros, which it leaves zero.

    ``score_out`` fp32 / ``logit_out`` (the logits' dtype) [M, B, V], each optional (generate's ``output_scores`` /
    ``output_logits``): a row that is not finished, with gen[b] < M, writes its score row (``score_rows``) and its logits
    to column gen[b].  Other columns are left alone."""
    B, V = logits.shape
    if logits.is_cuda and logits.dtype == torch.bfloat16 and _lib.has_symbol("odb_dec_sample"):
        assert logits.stride(1) == 1 and V <= MAX_SAMPLE_VOCAB and out.is_contiguous()
        if hist is not None:
            assert hist.dtype == torch.int32 and hist.is_contiguous() and hist.shape[0] == B
            assert scratch is not None and scratch.is_contiguous() and scratch.numel() >= B * 2 * ((V + 31) // 32)
        tab = table is not None and hist is not None
        if tab:
            assert seq_scratch is not None and seq_scratch.dtype == torch.float32 and seq_scratch.is_contiguous()
            assert seq_scratch.numel() >= B * V
        cols = _check_outputs(score_out, logit_out, B, V)
        _lib.check(_lib.cuda_lib().odb_dec_sample(logits.data_ptr(), logits.stride(0), V, ictl.data_ptr(), fctl.data_ptr(), pos.data_ptr(),
                                                  gen.data_ptr(), finished.data_ptr(), out.data_ptr(), out.shape[1],
                                                  ids_next.data_ptr(), hist.data_ptr() if hist is not None else None,
                                                  hist.shape[1] if hist is not None else 0,
                                                  scratch.data_ptr() if hist is not None else None,
                                                  table.ints.data_ptr() if tab else None, table.bias.data_ptr() if tab else None,
                                                  seq_scratch.data_ptr() if tab else None, _ptr(score_out), _ptr(logit_out), cols,
                                                  B, _lib.stream_ptr(logits)),
                   "dec_sample")
        _lib.count_launch()
        return
    c = ictl.tolist()
    fc = fctl.tolist()
    temperature, top_p, min_p = fc[FCTL_TEMPERATURE], fc[FCTL_TOP_P], fc[FCTL_MIN_P]
    x = logits.float()
    proc = hist is not None and processors_on(c, fc)
    if proc:
        x = process_logits_reference(x, hist, pos.long() + 1, gen, fc[FCTL_PENALTY], c[CTL_NGRAM], c[CTL_MIN_NEW],
                                     c[CTL_EOS:CTL_EOS + c[CTL_N_EOS]], _table_entries(table, c), c[CTL_MIN_LEN])
    tok = x.argmax(dim=-1)
    if c[CTL_DO_SAMPLE] and c[CTL_TOP_K] != 1:
        if proc:
            ok = torch.isfinite(x.max(dim=-1).values)
            drawn = _sample_reference(torch.where(ok[:, None], x, torch.zeros_like(x)), temperature, c[CTL_TOP_K], top_p, c[CTL_SEED],
                                      int(gen.min()), min_p)
            tok = torch.where(ok, drawn, tok)
        else:
            tok = _sample_reference(x, temperature, c[CTL_TOP_K], top_p, c[CTL_SEED], int(gen.min()), min_p)
    fin = finished.bool()
    g = gen.long()
    rows = torch.arange(B, device=logits.device)
    if score_out is not None or logit_out is not None:
        live = ~fin & (g < (score_out if score_out is not None else logit_out).shape[0])
        if score_out is not None:
            score_out[g[live], rows[live]] = score_rows(x, c, fc)[live].to(score_out.device)
        if logit_out is not None:
            logit_out[g[live], rows[live]] = logits[live]
    tok = torch.where(fin, torch.full_like(tok, c[CTL_PAD]), tok)
    inside = g < out.shape[1]
    out[rows[inside], g[inside]] = tok[inside]
    ids_next.copy_(tok)
    if hist is not None:
        at = pos.long().to(hist.device) + 1
        ok = at < hist.shape[1]
        hist[torch.arange(B, device=hist.device)[ok], at[ok]] = tok.to(hist.device, hist.dtype)[ok]
    gen.add_(1)
    pos.add_(1)
    eos = torch.tensor(c[CTL_EOS:CTL_EOS + c[CTL_N_EOS]], dtype=torch.int64, device=logits.device)
    finished.copy_((fin | torch.isin(tok, eos)).to(finished.dtype))


def score_rows(x: torch.Tensor, ictl: list[int], fctl: list[float]) -> torch.Tensor:
    """HF's score rows of the values x [rows, V] fp32 a sampler or an acceptance picks from (the logits after the logits
    processors): greedy, x itself; sampling, ``warp_logits`` (x / temperature, -inf outside the kept set); sampling with
    top_k = 1, x / temperature at the argmax alone (-inf elsewhere)."""
    if not ictl[CTL_DO_SAMPLE]:
        return x
    temperature = fctl[FCTL_TEMPERATURE]
    if ictl[CTL_TOP_K] == 1:
        top = x.argmax(dim=-1, keepdim=True)
        return torch.full_like(x, float("-inf")).scatter(-1, top, x.gather(-1, top) / temperature)
    return warp_logits(x, temperature, ictl[CTL_TOP_K], fctl[FCTL_TOP_P], fctl[FCTL_MIN_P])


def padding_rows(buf: torch.Tensor, pad: int) -> torch.Tensor:
    """Fills a score or logit buffer [..., V] with the padding row of generate's outputs: -inf everywhere, 0 at ``pad``
    (a column where a row had already finished)."""
    buf.fill_(float("-inf"))
    buf[..., pad] = 0.0
    return buf


def _check_outputs(score_out: torch.Tensor | None, logit_out: torch.Tensor | None, rows: int, V: int) -> int:
    """The kernels' score / logit buffers: contiguous [M, rows, V], fp32 / bf16, the same M; returns M (0: none)."""
    cols = 0
    for t, dt in ((score_out, torch.float32), (logit_out, torch.bfloat16)):
        if t is not None:
            assert t.dtype == dt and t.is_contiguous() and t.dim() == 3 and t.shape[1:] == (rows, V) and cols in (0, t.shape[0])
            cols = t.shape[0]
    return cols


def warp_logits(x: torch.Tensor, temperature: float, top_k: int, top_p: float, min_p: float = 0.0) -> torch.Tensor:
    """HF's logits warpers in HF's order (temperature, top-k, top-p, min-p) on fp32 logits [B, V]; removed entries are
    -inf.  Min-p (> 0) removes the tokens whose probability is below min_p times the largest one (never the largest)."""
    x = x / temperature
    if 0 < top_k < x.shape[-1]:
        kth = torch.topk(x, top_k, dim=-1).values[..., -1:]
        x = x.masked_fill(x < kth, float("-inf"))
    if top_p < 1.0:
        srt, idx = torch.sort(x, descending=False, dim=-1)
        cum = srt.softmax(dim=-1).cumsum(dim=-1)
        remove = cum <= (1 - top_p)
        remove[..., -1:] = False
        x = x.masked_fill(remove.scatter(-1, idx, remove), float("-inf"))
    if min_p > 0:
        probs = torch.softmax(x, dim=-1)
        remove = probs < min_p * probs.amax(dim=-1, keepdim=True)
        remove.scatter_(-1, torch.topk(probs, 1, dim=-1).indices, False)
        x = x.masked_fill(remove, float("-inf"))
    return x


def _sample_reference(x: torch.Tensor, temperature: float, top_k: int, top_p: float, seed: int, step: int,
                      min_p: float = 0.0) -> torch.Tensor:
    probs = torch.softmax(warp_logits(x, temperature, top_k, top_p, min_p), dim=-1)
    gen = torch.Generator(device=x.device).manual_seed((int(seed) * 1000003 + int(step)) & ((1 << 63) - 1))
    return torch.multinomial(probs, 1, generator=gen)[:, 0]
