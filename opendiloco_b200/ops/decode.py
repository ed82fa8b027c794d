"""Front-ends of the decode kernels (``csrc/decode_sm90.cu``) with a PyTorch reference beside each.

Dispatch follows :mod:`opendiloco_b200.ops.kernels`: tensors that qualify for the kernels (``usable``: CUDA, bf16,
head_dim 64, library symbols present) run our kernels; everything else (CPU, fp32, fp16) runs the reference, which is
also the test oracle.

KV cache layout, per layer: K and V each ``[B, Hkv, Smax, D]`` in the compute dtype.  ``pos`` (int32 ``[B]``) is the
position of each row's current token: ``rope_append`` writes at ``pos[b]`` and ``attention`` attends to keys
``0 .. pos[b]``; the sampler advances it.

Assisted generation scores n tokens per row in one pass.  Its buffers are slot-major: row ``j*B + b`` is token j of row
b, at position ``pos[b] + j`` (``rope_append_multi``, ``verify_attention``, ``accept``).
"""
from __future__ import annotations

import ctypes
import math

import torch

from .. import _lib

c_void_p, c_int, c_ll, c_float = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_float
_lib.register_optional("odb_dec_rope_append", [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                               c_int, c_void_p])
_lib.register_optional("odb_dec_kv_fill", [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p])
_lib.register_optional("odb_dec_attn_chunks", [c_int])
_lib.register_optional("odb_dec_attn", [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int, c_int,
                                        c_int, c_int, c_float, c_void_p])
_lib.register_optional("odb_dec_sample", [c_void_p, c_ll, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                          c_void_p, c_int, c_void_p])
_lib.register_optional("odb_dec_rope_append_multi", [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                                     c_int, c_int, c_int, c_void_p])
_lib.register_optional("odb_dec_verify_attn", [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_ll, c_int,
                                               c_int, c_int, c_int, c_int, c_float, c_void_p])
_lib.register_optional("odb_dec_accept", [c_void_p, c_ll, c_void_p, c_ll, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p])

MAX_EOS = 8
# int64 control block of the sampler: do_sample, top_k, seed, pad_token_id, n_eos, eos ids
CTL_DO_SAMPLE, CTL_TOP_K, CTL_SEED, CTL_PAD, CTL_N_EOS, CTL_EOS = range(6)
CTL_SIZE = CTL_EOS + MAX_EOS
MAX_SAMPLE_VOCAB = 56000          # the sampler keeps one fp32 per vocabulary entry in shared memory


def usable(t: torch.Tensor, head_dim: int, Hq: int = 1, Hkv: int = 1) -> bool:
    """Our decode kernels apply: CUDA bf16, head_dim 64, a GQA group of 1, 2, 4 or 8 query heads, symbols present."""
    return (t.is_cuda and t.dtype == torch.bfloat16 and head_dim == 64 and Hq % Hkv == 0 and Hq // Hkv in (1, 2, 4, 8)
            and _lib.has_symbol("odb_dec_attn") and _lib.has_symbol("odb_dec_sample"))


def usable_verify(t: torch.Tensor, head_dim: int, Hq: int = 1, Hkv: int = 1) -> bool:
    """``usable`` plus the assisted-generation kernels (multi-token RoPE+append, verify attention, acceptance)."""
    return (usable(t, head_dim, Hq, Hkv) and _lib.has_symbol("odb_dec_verify_attn") and _lib.has_symbol("odb_dec_accept")
            and _lib.has_symbol("odb_dec_rope_append_multi"))


def verify_splits(Smax: int) -> int:
    """Key tiles of 64 in a cache of Smax positions: the most splits ``verify_attention`` uses (sizes its partials)."""
    return (Smax + 63) // 64


def attn_chunks(Smax: int) -> int:
    return int(_lib.cuda_lib().odb_dec_attn_chunks(Smax))


# ------------------------------------------------------------------------------------------------ RoPE + append
def rope_append(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, pos: torch.Tensor, kc: torch.Tensor, vc: torch.Tensor,
                Hq: int, Hkv: int, D: int) -> None:
    """qkv [B, (Hq+2*Hkv)*D] (one token per row): rotate q (in place) and k at position pos[b]; k, v -> cache[b, :, pos[b]]."""
    B = qkv.shape[0]
    Smax = kc.shape[2]
    if usable(qkv, D, Hq, Hkv):
        assert qkv.stride(1) == 1 and kc.is_contiguous() and vc.is_contiguous() and pos.dtype == torch.int32
        _lib.check(_lib.cuda_lib().odb_dec_rope_append(qkv.data_ptr(), qkv.stride(0), cos.data_ptr(), sin.data_ptr(), pos.data_ptr(),
                                                       kc.data_ptr(), vc.data_ptr(), B, Hq, Hkv, Smax, _lib.stream_ptr(qkv)),
                   "dec_rope_append")
        _lib.count_launch()
        return
    half = D // 2
    p = pos.long()
    c, s = cos[p][:, None, :], sin[p][:, None, :]                     # [B, 1, D/2]
    x = qkv[:, : (Hq + Hkv) * D].float().view(B, Hq + Hkv, D)
    a, b = x[..., :half], x[..., half:]
    rot = torch.cat([a * c - b * s, b * c + a * s], dim=-1).to(qkv.dtype)
    qkv[:, : Hq * D] = rot[:, :Hq].reshape(B, Hq * D)
    rows = torch.arange(B, device=qkv.device)
    kc[rows, :, p] = rot[:, Hq:]
    vc[rows, :, p] = qkv[:, (Hq + Hkv) * D:].view(B, Hkv, D)


def kv_fill(qkv: torch.Tensor, lens: torch.Tensor, kc: torch.Tensor, vc: torch.Tensor, B: int, Sp: int, Hq: int, Hkv: int,
            D: int) -> None:
    """Prefill: rows s < lens[b] of the rotated packed projections qkv [B*Sp, row] -> cache[b, :, s]."""
    Smax = kc.shape[2]
    if usable(qkv, D, Hq, Hkv):
        assert qkv.stride(1) == 1 and kc.is_contiguous() and vc.is_contiguous() and lens.dtype == torch.int32
        _lib.check(_lib.cuda_lib().odb_dec_kv_fill(qkv.data_ptr(), qkv.stride(0), lens.data_ptr(), kc.data_ptr(), vc.data_ptr(), B, Sp,
                                                   Hq, Hkv, Smax, _lib.stream_ptr(qkv)), "dec_kv_fill")
        _lib.count_launch()
        return
    n = min(Sp, Smax)
    rows = qkv.view(B, Sp, -1)[:, :n]
    k = rows[..., Hq * D:(Hq + Hkv) * D].unflatten(-1, (Hkv, D)).transpose(1, 2)     # [B, Hkv, n, D]
    v = rows[..., (Hq + Hkv) * D:].unflatten(-1, (Hkv, D)).transpose(1, 2)
    keep = (torch.arange(n, device=qkv.device)[None, :] < lens.long()[:, None].to(qkv.device))[:, None, :, None]
    kc[:, :, :n] = torch.where(keep, k, kc[:, :, :n])
    vc[:, :, :n] = torch.where(keep, v, vc[:, :, :n])


# ------------------------------------------------------------------------------------------------ decode attention
def attention(q: torch.Tensor, kc: torch.Tensor, vc: torch.Tensor, pos: torch.Tensor, out: torch.Tensor, Hq: int, Hkv: int, D: int,
              part_o: torch.Tensor | None = None, part_ml: torch.Tensor | None = None) -> torch.Tensor:
    """out[b, h*D:(h+1)*D] = softmax(q_bh . K[b, h//G, :pos[b]+1]^T / sqrt(D)) V[b, h//G, :pos[b]+1]  (one query per row).

    q: the first Hq*D columns of [B, row].  part_o fp32 [B, Hq, chunks, D] / part_ml fp32 [B, Hq, chunks, 2]: scratch of
    the split-KV kernel (``attn_chunks(Smax)`` chunks)."""
    B = q.shape[0]
    Smax = kc.shape[2]
    if usable(q, D, Hq, Hkv):
        assert q.stride(1) == 1 and out.stride(1) == 1 and kc.is_contiguous() and vc.is_contiguous() and pos.dtype == torch.int32
        _lib.check(_lib.cuda_lib().odb_dec_attn(q.data_ptr(), q.stride(0), kc.data_ptr(), vc.data_ptr(), pos.data_ptr(), part_o.data_ptr(),
                                                part_ml.data_ptr(), out.data_ptr(), out.stride(0), B, Hq, Hkv, Smax,
                                                1.0 / math.sqrt(D), _lib.stream_ptr(q)), "dec_attn")
        _lib.count_launch(2)
        return out
    G = Hq // Hkv
    qf = q[:, : Hq * D].float().view(B, Hkv, G, D)
    att = torch.einsum("bkgd,bksd->bkgs", qf, kc.float()) / math.sqrt(D)
    valid = torch.arange(Smax, device=q.device)[None, :] <= pos.long().to(q.device)[:, None]
    att = att.masked_fill(~valid[:, None, None, :], float("-inf"))
    o = torch.einsum("bkgs,bksd->bkgd", torch.softmax(att, dim=-1), vc.float())
    out.copy_(o.reshape(B, Hq * D).to(out.dtype))
    return out


# ------------------------------------------------------------------------------------------------ assisted generation
def rope_append_multi(qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, pos: torch.Tensor, kc: torch.Tensor, vc: torch.Tensor,
                      Hq: int, Hkv: int, D: int, n: int) -> None:
    """qkv [n*B, row] slot-major: rotate q (in place) and k of row j*B + b at position pos[b] + j; k, v -> cache[b, :, pos[b] + j]."""
    B = qkv.shape[0] // n
    Smax = kc.shape[2]
    if usable_verify(qkv, D, Hq, Hkv):
        assert qkv.stride(1) == 1 and kc.is_contiguous() and vc.is_contiguous() and pos.dtype == torch.int32
        _lib.check(_lib.cuda_lib().odb_dec_rope_append_multi(qkv.data_ptr(), qkv.stride(0), cos.data_ptr(), sin.data_ptr(),
                                                             pos.data_ptr(), kc.data_ptr(), vc.data_ptr(), B, n, Hq, Hkv, Smax,
                                                             _lib.stream_ptr(qkv)), "dec_rope_append_multi")
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
    kc[rows, :, p] = rot[:, Hq:]
    vc[rows, :, p] = qkv[:, (Hq + Hkv) * D:].view(n * B, Hkv, D)


def verify_attention(q: torch.Tensor, kc: torch.Tensor, vc: torch.Tensor, pos: torch.Tensor, out: torch.Tensor, Hq: int, Hkv: int,
                     D: int, n: int, part_o: torch.Tensor | None = None, part_ml: torch.Tensor | None = None) -> torch.Tensor:
    """Attention of n queries per row, slot-major: query row j*B + b attends keys 0 .. pos[b] + j of row b (causal inside
    the block).  part_o fp32 [n*B, Hq, verify_splits(Smax), D] / part_ml fp32 [n*B, Hq, verify_splits(Smax), 2]: scratch
    of the split-KV kernel."""
    B = q.shape[0] // n
    Smax = kc.shape[2]
    if usable_verify(q, D, Hq, Hkv):
        assert n <= 8 and q.stride(1) == 1 and out.stride(1) == 1 and kc.is_contiguous() and vc.is_contiguous()
        assert pos.dtype == torch.int32 and part_o.shape[2] == verify_splits(Smax) and part_ml.shape[2] == verify_splits(Smax)
        _lib.check(_lib.cuda_lib().odb_dec_verify_attn(q.data_ptr(), q.stride(0), kc.data_ptr(), vc.data_ptr(), pos.data_ptr(),
                                                       part_o.data_ptr(), part_ml.data_ptr(), out.data_ptr(), out.stride(0), B, n, Hq,
                                                       Hkv, Smax, 1.0 / math.sqrt(D), _lib.stream_ptr(q)), "dec_verify_attn")
        _lib.count_launch(2)
        return out
    G = Hq // Hkv
    qf = q[:, : Hq * D].float().view(n, B, Hkv, G, D)
    att = torch.einsum("jbkgd,bksd->jbkgs", qf, kc.float()) / math.sqrt(D)
    last = pos.long().to(q.device)[None, :] + torch.arange(n, device=q.device)[:, None]                   # [n, B]
    valid = torch.arange(Smax, device=q.device)[None, None, :] <= last[:, :, None]
    att = att.masked_fill(~valid[:, :, None, None, :], float("-inf"))
    o = torch.einsum("jbkgs,bksd->jbkgd", torch.softmax(att, dim=-1), vc.float())
    out.copy_(o.reshape(n * B, Hq * D).to(out.dtype))
    return out


def accept(plog: torch.Tensor, qlog: torch.Tensor, ictl: torch.Tensor, fctl: torch.Tensor, tok: torch.Tensor, pos: torch.Tensor,
           gen: torch.Tensor, finished: torch.Tensor, out: torch.Tensor, max_new: int, draft_pos: torch.Tensor,
           stats: torch.Tensor) -> None:
    """The acceptance step of one assisted round (speculative sampling; Leviathan et al. 2023, Chen et al. 2023).

    plog [(K+1)*B, V]: the target's logits, slot-major, slot i predicting the token at pos[b] + i + 1; qlog [K*B, V]: the
    draft's logits for its proposals; tok [(K+1)*B]: slot 0 the row's last token, slots 1..K the proposals d_1..d_K.

    Greedy (ictl do_sample = 0, or top_k = 1): accept the longest prefix where d_i is the target's argmax, then emit the
    argmax at the first mismatch (or the bonus argmax after d_K).  Sampling: p and q are both distributions after the
    sampler's warpers; d_i is accepted with probability min(1, p(d_i) / q(d_i)); the first rejection draws from
    normalise(max(0, p - q)); K acceptances draw the bonus token from p_{K+1}.

    The emitted tokens go to out[b, gen[b]..] (a row stops after an EOS id or at max_new tokens; later tokens are never
    written), gen / pos / finished advance (a row that finishes keeps its pos), tok slot 0 becomes the next round's last
    token and draft_pos = pos.  Finished rows are left alone.  stats int64 [B, 2] += (1, accepted proposals) per row that
    took part.  CUDA draws use Philox keyed by (seed, row, gen[b], slot); the reference draws from a torch generator
    seeded by (seed, row, gen[b]), so the paths give different (equally distributed) samples for the same seed."""
    B = pos.shape[0]
    K = qlog.shape[0] // B
    V = plog.shape[1]
    if plog.is_cuda and plog.dtype == torch.bfloat16 and _lib.has_symbol("odb_dec_accept"):
        assert plog.stride(1) == 1 and qlog.stride(1) == 1 and V <= MAX_SAMPLE_VOCAB and out.is_contiguous() and 1 <= K <= 7
        _lib.check(_lib.cuda_lib().odb_dec_accept(plog.data_ptr(), plog.stride(0), qlog.data_ptr(), qlog.stride(0), V, K, ictl.data_ptr(),
                                                  fctl.data_ptr(), tok.data_ptr(), pos.data_ptr(), gen.data_ptr(), finished.data_ptr(),
                                                  out.data_ptr(), out.shape[1], max_new, draft_pos.data_ptr(), stats.data_ptr(), B,
                                                  _lib.stream_ptr(plog)), "dec_accept")
        _lib.count_launch()
        return
    c = ictl.tolist()
    temperature, top_p = (float(v) for v in fctl.tolist())
    greedy = not (c[CTL_DO_SAMPLE] and c[CTL_TOP_K] != 1)
    eos = set(c[CTL_EOS:CTL_EOS + c[CTL_N_EOS]])
    p_all = plog.float().view(K + 1, B, V)
    q_all = qlog.float().view(K, B, V)
    t = tok.view(K + 1, B)
    for b in range(B):
        if finished[b]:
            draft_pos[b] = pos[b]
            continue
        g0 = int(gen[b])
        drafts = [int(t[i + 1, b]) for i in range(K)]
        n_acc, t_new = 0, 0
        if greedy:
            am = p_all[:, b].argmax(dim=-1).tolist()
            while n_acc < K and drafts[n_acc] == am[n_acc]:
                n_acc += 1
            t_new = am[n_acc]
        else:
            rng = torch.Generator(device="cpu").manual_seed((int(c[CTL_SEED]) * 1000003 + b * 7919 + g0) & ((1 << 63) - 1))
            p = torch.softmax(warp_logits(p_all[:, b].cpu(), temperature, c[CTL_TOP_K], top_p), dim=-1)          # [K+1, V]
            q = torch.softmax(warp_logits(q_all[:, b].cpu(), temperature, c[CTL_TOP_K], top_p), dim=-1)          # [K, V]
            while n_acc < K:
                d = drafts[n_acc]
                u = float(torch.rand((), generator=rng))
                if p[n_acc, d] > 0 and u * q[n_acc, d] <= p[n_acc, d]:
                    n_acc += 1
                    continue
                res = (p[n_acc] - q[n_acc]).clamp(min=0)
                t_new = int(torch.multinomial(res if float(res.sum()) > 0 else p[n_acc], 1, generator=rng))
                break
            else:
                t_new = int(torch.multinomial(p[K], 1, generator=rng))
        g, fin = g0, False
        for x in drafts[:n_acc] + [t_new]:
            if fin or g >= max_new:
                break
            out[b, g] = x
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
        draft_pos[b] = pos[b]


# ------------------------------------------------------------------------------------------------ sampler
def make_controls(do_sample: bool, temperature: float, top_k: int, top_p: float, seed: int, pad: int, eos: list[int], device):
    """(ictl int64 [CTL_SIZE], fctl fp32 [2]) for ``sample``."""
    if len(eos) > MAX_EOS:
        raise ValueError(f"at most {MAX_EOS} EOS ids are supported, got {len(eos)}")
    ictl = [int(do_sample), int(top_k), int(seed) & ((1 << 63) - 1), int(pad), len(eos)] + list(eos) + [0] * (MAX_EOS - len(eos))
    return (torch.tensor(ictl, dtype=torch.int64, device=device),
            torch.tensor([float(temperature), float(top_p)], dtype=torch.float32, device=device))


def sample(logits: torch.Tensor, ictl: torch.Tensor, fctl: torch.Tensor, pos: torch.Tensor, gen: torch.Tensor, finished: torch.Tensor,
           out: torch.Tensor, ids_next: torch.Tensor) -> None:
    """Pick one token per row of logits [B, V] and write it to out[b, gen[b]] and ids_next[b]; then gen += 1, pos += 1.

    Greedy (ictl do_sample = 0, or top_k = 1): argmax, ties to the lowest index.  Sampling: logits / temperature, keep the
    top_k largest (0 = all; ties with the k-th value are kept), keep the smallest set of largest probabilities whose mass
    reaches top_p (every token tied with the smallest kept one is kept too), draw from the rest.  A row that has produced an EOS id emits ``pad`` from then on (``finished``).
    CUDA draws use Philox keyed by (seed, row, gen[b]); the reference draws from a torch generator seeded by (seed, step),
    so the two paths give different (equally distributed) samples for the same seed."""
    B, V = logits.shape
    if logits.is_cuda and logits.dtype == torch.bfloat16 and _lib.has_symbol("odb_dec_sample"):
        assert logits.stride(1) == 1 and V <= MAX_SAMPLE_VOCAB and out.is_contiguous()
        _lib.check(_lib.cuda_lib().odb_dec_sample(logits.data_ptr(), logits.stride(0), V, ictl.data_ptr(), fctl.data_ptr(), pos.data_ptr(),
                                                  gen.data_ptr(), finished.data_ptr(), out.data_ptr(), out.shape[1],
                                                  ids_next.data_ptr(), B, _lib.stream_ptr(logits)), "dec_sample")
        _lib.count_launch()
        return
    c = ictl.tolist()
    temperature, top_p = (float(v) for v in fctl.tolist())
    x = logits.float()
    tok = x.argmax(dim=-1)
    if c[CTL_DO_SAMPLE] and c[CTL_TOP_K] != 1:
        tok = _sample_reference(x, temperature, c[CTL_TOP_K], top_p, c[CTL_SEED], int(gen.min()))
    fin = finished.bool()
    tok = torch.where(fin, torch.full_like(tok, c[CTL_PAD]), tok)
    g = gen.long()
    rows = torch.arange(B, device=logits.device)
    inside = g < out.shape[1]
    out[rows[inside], g[inside]] = tok[inside]
    ids_next.copy_(tok)
    gen.add_(1)
    pos.add_(1)
    eos = torch.tensor(c[CTL_EOS:CTL_EOS + c[CTL_N_EOS]], dtype=torch.int64, device=logits.device)
    finished.copy_((fin | torch.isin(tok, eos)).to(finished.dtype))


def warp_logits(x: torch.Tensor, temperature: float, top_k: int, top_p: float) -> torch.Tensor:
    """HF's logits warpers in HF's order (temperature, top-k, top-p) on fp32 logits [B, V]; removed entries are -inf."""
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
    return x


def _sample_reference(x: torch.Tensor, temperature: float, top_k: int, top_p: float, seed: int, step: int) -> torch.Tensor:
    probs = torch.softmax(warp_logits(x, temperature, top_k, top_p), dim=-1)
    gen = torch.Generator(device=x.device).manual_seed((int(seed) * 1000003 + int(step)) & ((1 << 63) - 1))
    return torch.multinomial(probs, 1, generator=gen)[:, 0]
