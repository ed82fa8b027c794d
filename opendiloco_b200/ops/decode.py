"""Front-ends of the decode kernels (``csrc/decode_sm90.cu``) with a PyTorch reference beside each.

Dispatch follows :mod:`opendiloco_b200.ops.kernels`: tensors that qualify for the kernels (``usable``: CUDA, bf16,
head_dim 64, library symbols present) run our kernels; everything else (CPU, fp32, fp16) runs the reference, which is
also the test oracle.

KV cache layout, per layer: K and V each ``[B, Hkv, Smax, D]`` in the compute dtype.  ``pos`` (int32 ``[B]``) is the
position of each row's current token: ``rope_append`` writes at ``pos[b]`` and ``attention`` attends to keys
``0 .. pos[b]``; the sampler advances it.
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

MAX_EOS = 8
# int64 control block of the sampler: do_sample, top_k, seed, pad_token_id, n_eos, eos ids
CTL_DO_SAMPLE, CTL_TOP_K, CTL_SEED, CTL_PAD, CTL_N_EOS, CTL_EOS = range(6)
CTL_SIZE = CTL_EOS + MAX_EOS
MAX_SAMPLE_VOCAB = 56000          # the sampler keeps one fp32 per vocabulary entry in shared memory


def usable(t: torch.Tensor, head_dim: int, Hq: int = 1, Hkv: int = 1) -> bool:
    """Our decode kernels apply: CUDA bf16, head_dim 64, a GQA group of 1, 2, 4 or 8 query heads, symbols present."""
    return (t.is_cuda and t.dtype == torch.bfloat16 and head_dim == 64 and Hq % Hkv == 0 and Hq // Hkv in (1, 2, 4, 8)
            and _lib.has_symbol("odb_dec_attn") and _lib.has_symbol("odb_dec_sample"))


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
