"""Row-by-row oracle for the sm_90a attention kernels: the training forward / backward (csrc/attn_sm90.cu,
csrc/attn_bwd_sm90.cu), split-KV decode attention and multi-query verify attention (csrc/decode_sm90.cu), each against
an independent float64 reference written here, fed the same bf16 values the kernel reads.

Inputs come in five regimes, because random inputs leave the softmax almost flat:
  uniform    q, k, v ~ N(0, 1): scaled scores have std ~1
  peaked     q, k ~ N(0, 9): scaled scores have std ~9, rows dominated by a handful of keys
  sink       key 0 of every sequence is aligned with every query: most of the mass sits on token 0
  late_max   the score grows by SLOPE nats per key index, so each row's maximum lies in its last (diagonal) key tile and
             the running max moves by ~3 nats per 64-key tile; split-K chunk maxima differ by up to ~100 nats
  zero_q     even query heads have q = 0: out is the running mean of v and lse = log(s + 1), exactly

Every (batch, head, position) row gets its own error (``_row_err``).  In every tile of positions (64 queries or keys in
training, one row in decode, the n queries of a row in verify) the worst row must stay within ``c x (the worst row of
torch's own bf16 SDPA in the same tile, same inputs) + floor``; a failure names the tile and the worst row.  lse is
checked per element against float64.
"""
import math

import pytest
import torch
import torch.nn.functional as F
from torch.nn.attention import SDPBackend, sdpa_kernel

from opendiloco_b200.ops import attention as A
from opendiloco_b200.ops import decode as DK
from opendiloco_b200.ops import kernels as K

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
D = 64
REGIMES = ["uniform", "peaked", "sink", "late_max", "zero_q"]
SLOPE = 0.05                       # late_max: nats of scaled score per key index

# (c, floor): in every tile of positions, worst row of ours <= c x worst row of torch bf16 + floor (``_assert_rows``).
# Measured on an H100 80GB HBM3 (700 W), torch 2.11, over every case below: the largest ratio ours / torch of a tile,
# and the floor a bound with c = 1 would need (the largest excess of ours over torch in a tile).
BOUND = {
    "out": (1.5, 1e-3),            # ratio 1.23, excess 6.3e-4; worst row 3.9e-3 (torch 3.9e-3)
    "dq": (3.0, 2e-2),             # ratio 3.12 (late_max), excess at c = 3: 1.2e-2; worst row 2.6 (torch 2.6, sink:
                                   # D = rowsum(dO * O) from the bf16 O nearly cancels, times |k_0| = 24)
    "dk": (3.0, 2e-3),             # ratio 2.89 (peaked), excess at c = 3: none; worst row 0.34 (torch 0.34)
    "dv": (1.5, 1e-3),             # ratio 1.28, excess 8.5e-4; worst row 4.9e-3 (torch 5.3e-3)
    "decode": (1.5, 0.0),          # ratio <= 1.0 (excess 1.5e-7); worst row 2.7e-3 (torch 3.2e-3)
    "verify": (1.5, 1e-3),         # ratio 1.27, excess 5.9e-4; worst row 3.5e-3 (torch 3.5e-3)
}


# ------------------------------------------------------------------------------------------------ inputs
def _inputs(regime, B, Hq, Hkv, Sq, Sk, seed):
    """bf16 q [B, Hq, Sq, D], k / v [B, Hkv, Sk, D]; key index = position in the sequence (or in the cache)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    q = torch.randn(B, Hq, Sq, D, device=DEV, generator=g)
    k = torch.randn(B, Hkv, Sk, D, device=DEV, generator=g)
    v = torch.randn(B, Hkv, Sk, D, device=DEV, generator=g)
    if regime == "peaked":
        q *= 3.0
        k *= 3.0
    elif regime == "sink":
        q[..., 0] += 4.0                         # q . k_0 / 8 = 3 q_0 ~ N(12, 3^2) against N(0, ~1.25) for the rest
        k[:, :, 0, 0] = 24.0
    elif regime == "late_max":
        q[..., 0] = 4.0                          # q . k_j / 8 = SLOPE * j + N(0, ~1)
        k[..., 0] = torch.arange(Sk, device=DEV, dtype=torch.float32) * (8.0 * SLOPE / 4.0)
    elif regime == "zero_q":
        q[:, ::2] = 0.0
    else:
        assert regime == "uniform", regime
    return q.to(BF), k.to(BF), v.to(BF)


def _tokens(x):
    """[B, H, S, D] -> token-major [B*S, H*D]."""
    B, H, S, _ = x.shape
    return x.permute(0, 2, 1, 3).reshape(B * S, H * D)


def _heads(x, B, S, H):
    """token-major [B*S, H*D] -> [B, H, S, D] (a view)."""
    return x.view(B, S, H, D).permute(0, 2, 1, 3)


# ------------------------------------------------------------------------------------------------ float64 reference
def _reference(q, k, v, qpos, dout=None):
    """One batch row in float64: q [Hq, Sq, D], k / v [Hkv, Sk, D]; query i sits at position qpos[i] and sees keys
    0 .. qpos[i]; query head h reads kv head h // (Hq // Hkv) (the HF GQA mapping); scale 1/sqrt(D).  Returns out
    [Hq, Sq, D], lse [Hq, Sq] (natural log) and, given dout, (dq, dk, dv) through float64 autograd."""
    G = q.shape[0] // k.shape[0]
    grad = dout is not None
    q, k, v = (t.detach().double().requires_grad_(grad) for t in (q, k, v))
    kk, vv = k.repeat_interleave(G, 0), v.repeat_interleave(G, 0)
    s = torch.einsum("hqd,hkd->hqk", q, kk) / math.sqrt(D)
    seen = torch.arange(k.shape[1], device=q.device)[None, :] <= qpos[:, None]
    s = s.masked_fill(~seen, float("-inf"))
    lse = torch.logsumexp(s, dim=-1)
    out = torch.einsum("hqk,hkd->hqd", torch.exp(s - lse[..., None]), vv)
    if not grad:
        return out.detach(), lse.detach(), None
    grads = torch.autograd.grad(out, (q, k, v), dout.double())
    return out.detach(), lse.detach(), grads


def _reference_batch(q, k, v, qpos, dout=None):
    """_reference over the batch rows (one at a time keeps the [Hq, Sq, Sk] float64 scores a few GB at most);
    qpos [B, Sq]."""
    rows = [_reference(q[b], k[b], v[b], qpos[b], None if dout is None else dout[b]) for b in range(q.shape[0])]
    out, lse = torch.stack([r[0] for r in rows]), torch.stack([r[1] for r in rows])
    grads = None if dout is None else tuple(torch.stack([r[2][i] for r in rows]) for i in range(3))
    return out, lse, grads


def _check_zero_q_reference(out_r, lse_r, v, qpos):
    """The closed form of the zero_q heads: out = mean of v over the keys seen, lse = log(number of keys seen)."""
    G = out_r.shape[1] // v.shape[1]
    cnt = (qpos + 1).double()                                                 # [B, Sq]
    mean = v.double().cumsum(2) / torch.arange(1, v.shape[2] + 1, device=DEV, dtype=torch.float64)[:, None]
    idx = qpos[:, None, :, None].expand(-1, v.shape[1], -1, D)
    mean = torch.gather(mean, 2, idx).repeat_interleave(G, 1)                 # [B, Hq, Sq, D]
    assert torch.allclose(out_r[:, ::2], mean[:, ::2], rtol=0, atol=1e-9)
    assert torch.allclose(lse_r[:, ::2], cnt.log()[:, None].expand_as(lse_r[:, ::2]), rtol=0, atol=1e-9)


# ------------------------------------------------------------------------------------------------ torch bf16 yardstick
def _torch_causal(q, k, v, dout):
    """torch's bf16 SDPA (flash or cuDNN) with autograd: the kv heads enter expanded to one per query head, and the
    group sum of their gradients is taken in fp32 and rounded once."""
    Hkv = k.shape[1]
    G = q.shape[1] // Hkv
    qq = q.detach().clone().requires_grad_()
    kk = k.detach().repeat_interleave(G, 1).requires_grad_()
    vv = v.detach().repeat_interleave(G, 1).requires_grad_()
    with sdpa_kernel([SDPBackend.FLASH_ATTENTION, SDPBackend.CUDNN_ATTENTION]):
        o = F.scaled_dot_product_attention(qq, kk, vv, is_causal=True)
        o.backward(dout)
    fold = lambda t: t.float().unflatten(1, (Hkv, G)).sum(2).to(BF)          # noqa: E731
    return o.detach(), qq.grad, fold(kk.grad), fold(vv.grad)


def _torch_masked(q, k, v, qpos):
    """torch's bf16 memory-efficient SDPA, query i of row b seeing keys 0 .. qpos[b, i] (decode and verify)."""
    G = q.shape[1] // k.shape[1]
    seen = torch.arange(k.shape[2], device=DEV)[None, None, :] <= qpos[:, :, None]
    with sdpa_kernel([SDPBackend.EFFICIENT_ATTENTION]):
        return F.scaled_dot_product_attention(q, k.repeat_interleave(G, 1), v.repeat_interleave(G, 1), attn_mask=seen[:, None])


# ------------------------------------------------------------------------------------------------ metric
def _row_err(x, ref):
    """Error of each row (last dim) of x against the float64 ref: |x - ref| / max(|ref|, rms / 16), with rms the
    root-mean-square row norm of ref over the tensor, so a row that carries almost no signal is judged on the tensor's
    scale instead of its own."""
    ref = ref.double()
    n = ref.norm(dim=-1)
    floor = float(n.square().mean().sqrt()) / 16
    return (x.double() - ref).norm(dim=-1) / n.clamp_min(floor)


def _worst(err):
    i = int(err.argmax())
    return float(err.view(-1)[i]), tuple(int(c) for c in torch.unravel_index(torch.tensor(i), err.shape))


def _assert_rows(case, pairs, tile):
    """pairs: name -> (ours [B, H, S, D], torch bf16, float64 reference).  The bound applies to every ``tile``
    consecutive positions of a head separately: the worst row of ours in the tile <= c x the worst row of torch in the
    same tile + floor.  Over the whole tensor that is the same bound on the worst row, but a tile with a wrong row cannot
    hide behind an ill-conditioned row elsewhere (dq rows whose D = rowsum(dO * O) nearly cancels carry relative errors
    near 1 in any bf16 implementation)."""
    line, failures = [case], []
    for name, (ours, theirs, ref) in pairs.items():
        c, floor = BOUND[name]
        e_ours, e_torch = _row_err(ours, ref), _row_err(theirs, ref)
        w_ours, where = _worst(e_ours)
        w_torch, _ = _worst(e_torch)
        B, H, S = e_ours.shape
        t_ours, t_torch = (e.view(B, H, S // tile, tile).amax(-1) for e in (e_ours, e_torch))
        excess, (b, h, t) = _worst(t_ours - (c * t_torch + floor))          # NaN ranks first
        ratio = float((t_ours / t_torch)[t_torch > 0].max())
        line.append(f"{name} {w_ours:.2e}@{where} (torch {w_torch:.2e}), tiles <= x{ratio:.2f} torch")
        if not excess <= 0:
            failures.append(f"{case}: {name} worst row of positions {t * tile}..{t * tile + tile - 1} of (b, h) = ({b}, {h}) "
                            f"is {float(t_ours[b, h, t]):.3e} > {c} x torch bf16 {float(t_torch[b, h, t]):.3e} + {floor:g} "
                            f"(worst row overall {w_ours:.3e} at (b, h, pos) = {where}, torch bf16 {w_torch:.3e})")
    print(" | ".join(line))
    assert not failures, "\n".join(failures)


def _assert_lse(case, lse, lse_ref):
    """lse per element: |ours - float64| <= 1e-3 + 1e-5 |lse|."""
    err = (lse.double() - lse_ref).abs()
    excess = err - (1e-3 + 1e-5 * lse_ref.abs())
    e, where = _worst(excess)
    print(f"{case} | lse max abs err {float(err.max()):.2e}")
    assert e <= 0, f"{case}: lse off by {float(err[where]):.3e} at (b, h, s) = {where} (ref {float(lse_ref[where]):.4f})"


# ------------------------------------------------------------------------------------------------ training fwd + bwd
def _unrope(x, cos, sin):
    """Rotation by -theta of the (j, j + D/2) pairs of x [B, H, S, D] in float64 (the transpose of RoPE)."""
    x = x.double()
    c, s = cos.double()[None, None], sin.double()[None, None]
    a, b = x[..., : D // 2], x[..., D // 2:]
    return torch.cat([a * c + b * s, b * c - a * s], dim=-1)


def _train_case(B, S, Hq, Hkv, regime, seed, pad=0, rope=False):
    case = f"train B{B} S{S} Hq{Hq} Hkv{Hkv} {regime}" + (f" pad{pad}" if pad else "") + (" packed+rope" if rope else "")
    q, k, v = _inputs(regime, B, Hq, Hkv, S, S, seed)
    row = (Hq + 2 * Hkv) * D
    qkv = torch.zeros(B * S, row + pad, dtype=BF, device=DEV)[:, :row]       # pad > 0: row stride wider than the row
    qkv.copy_(torch.cat([_tokens(q), _tokens(k), _tokens(v)], dim=1))
    out, lse = A.tc_attention_fwd(qkv, B, S, Hq, Hkv)
    dout = torch.randn(B * S, Hq * D, device=DEV, generator=torch.Generator(device=DEV).manual_seed(seed + 1)).to(BF)
    if rope:
        cos, sin = K.rope_tables(S, D, 10000.0, torch.device(DEV))
        packed = torch.zeros(B * S, row, dtype=BF, device=DEV)
        A.tc_attention_bwd(dout, qkv, out, lse, B, S, Hq, Hkv, dqkv=packed, cos=cos, sin=sin)
        dq, dk, dv = packed[:, : Hq * D], packed[:, Hq * D:(Hq + Hkv) * D], packed[:, (Hq + Hkv) * D:]
    else:
        dq, dk, dv = A.tc_attention_bwd(dout, qkv, out, lse, B, S, Hq, Hkv)
    torch.cuda.synchronize()

    dout_h = _heads(dout, B, S, Hq)
    qpos = torch.arange(S, device=DEV).expand(B, S)
    out_r, lse_r, (dq_r, dk_r, dv_r) = _reference_batch(q, k, v, qpos, dout_h)
    t_out, t_dq, t_dk, t_dv = _torch_causal(q, k, v, dout_h)
    if rope:
        dq_r, dk_r = _unrope(dq_r, cos, sin), _unrope(dk_r, cos, sin)
        t_dq, t_dk = _unrope(t_dq, cos, sin).to(BF), _unrope(t_dk, cos, sin).to(BF)
    if regime == "zero_q":
        _check_zero_q_reference(out_r, lse_r, v, qpos)

    _assert_lse(case, lse, lse_r)
    _assert_rows(case, {"out": (_heads(out, B, S, Hq), t_out, out_r), "dq": (_heads(dq, B, S, Hq), t_dq, dq_r),
                        "dk": (_heads(dk, B, S, Hkv), t_dk, dk_r), "dv": (_heads(dv, B, S, Hkv), t_dv, dv_r)}, tile=64)


# Every GQA group the kernels take, at one tile pair (S = 128), a query-tile count that is not a multiple of the
# backward's 128-key tile (384), and the longest context the configs allow (2048).  Group 32 is MQA (Hkv = 1).
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("group", [1, 2, 4, 8, 16, 32])
@pytest.mark.parametrize("S", [128, 384, 2048])
def test_train_attention_rows(S, group, regime):
    Hkv = 1 if group == 32 else 2
    B = {128: 3, 384: 2, 2048: 1}[S]
    _train_case(B, S, group * Hkv, Hkv, regime, seed=S * 100 + group * 7 + REGIMES.index(regime))


# The head layouts of the configs at their longest context: Llama-150M (16 heads) and Llama-1B (32 query heads, 4 kv).
@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("B,Hq,Hkv", [(4, 16, 16), (2, 32, 4)], ids=["150m", "1b"])
def test_train_attention_rows_model_layouts(B, Hq, Hkv, regime):
    _train_case(B, 2048, Hq, Hkv, regime, seed=Hq * 31 + REGIMES.index(regime))


@pytest.mark.parametrize("regime", ["uniform", "late_max"])
@pytest.mark.parametrize("pad", [8, 200])
def test_train_attention_rows_strided_qkv(pad, regime):
    """qkv is a column slice of a wider buffer: its row stride (row + pad elements) is not its row length."""
    _train_case(2, 384, 8, 2, regime, seed=pad + REGIMES.index(regime), pad=pad)


@pytest.mark.parametrize("regime", ["uniform", "sink", "late_max"])
def test_train_attention_rows_packed_rope(regime):
    """The packed dq|dk|dv output with the RoPE rotation undone by the kernels, against the float64 gradients rotated
    back in float64."""
    _train_case(2, 1024, 16, 4, regime, seed=77 + REGIMES.index(regime), rope=True)


# ------------------------------------------------------------------------------------------------ decode
DEC_SMAX = 2048
# lengths (pos + 1) on both sides of every 128-key chunk edge up to the end of the cache
DEC_LENGTHS = sorted({1, 2, DEC_SMAX - 1, DEC_SMAX} | {e + d for e in range(128, DEC_SMAX, 128) for d in (-1, 0, 1)})


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_decode_attention_rows(G, regime):
    Hkv, Smax, B = 2, DEC_SMAX, len(DEC_LENGTHS)
    Hq = G * Hkv
    case = f"decode G{G} Hq{Hq} Hkv{Hkv} {regime}"
    q, kc, vc = _inputs(regime, B, Hq, Hkv, 1, Smax, seed=1000 + G * 10 + REGIMES.index(regime))
    pos = torch.tensor(DEC_LENGTHS, dtype=torch.int32, device=DEV) - 1
    nch = DK.attn_chunks(Smax)
    part_o = torch.empty(B, Hq, nch, D, device=DEV)
    part_ml = torch.empty(B, Hq, nch, 2, device=DEV)
    out = torch.empty(B, Hq * D, dtype=BF, device=DEV)
    DK.attention(q[:, :, 0].reshape(B, Hq * D), kc, vc, pos, out, Hq, Hkv, D, part_o, part_ml)
    qpos = pos.long()[:, None]
    out_r, lse_r, _ = _reference_batch(q, kc, vc, qpos)
    if regime == "zero_q":
        _check_zero_q_reference(out_r, lse_r, vc, qpos)
    _assert_rows(case, {"decode": (out.view(B, Hq, 1, D), _torch_masked(q, kc, vc, qpos), out_r)}, tile=1)


# ------------------------------------------------------------------------------------------------ verify
VER_SMAX = 2048


def _verify_positions(n):
    """Slot-0 positions: the block ending at, straddling and starting at 64-key tile edges (320 and 384 are split
    edges at the batch size below), position 0 and the end of the cache."""
    ps = {0, VER_SMAX - n}
    for e in (64, 128, 320, 384, 1024, 1984):
        ps |= {e - n, e - 1, e}
    return sorted(p for p in ps if 0 <= p <= VER_SMAX - n)


@pytest.mark.parametrize("regime", REGIMES)
@pytest.mark.parametrize("n", [1, 2, 5, 8])
@pytest.mark.parametrize("G", [1, 2, 4, 8])
def test_verify_attention_rows(G, n, regime):
    Hkv, Smax = 2, VER_SMAX
    Hq = G * Hkv
    positions = _verify_positions(n)
    B = len(positions)
    case = f"verify G{G} n{n} Hq{Hq} Hkv{Hkv} B{B} {regime}"
    q, kc, vc = _inputs(regime, B, Hq, Hkv, n, Smax, seed=2000 + G * 100 + n * 10 + REGIMES.index(regime))
    pos = torch.tensor(positions, dtype=torch.int32, device=DEV)
    nsp = DK.verify_splits(Smax)
    part_o = torch.empty(n * B, Hq, nsp, D, device=DEV)
    part_ml = torch.empty(n * B, Hq, nsp, 2, device=DEV)
    out = torch.empty(n * B, Hq * D, dtype=BF, device=DEV)
    q_rows = q.permute(2, 0, 1, 3).reshape(n * B, Hq * D)                    # slot-major: row j*B + b
    DK.verify_attention(q_rows, kc, vc, pos, out, Hq, Hkv, D, n, part_o, part_ml)
    qpos = pos.long()[:, None] + torch.arange(n, device=DEV)[None, :]
    out_r, lse_r, _ = _reference_batch(q, kc, vc, qpos)
    if regime == "zero_q":
        _check_zero_q_reference(out_r, lse_r, vc, qpos)
    ours = out.view(n, B, Hq, D).permute(1, 2, 0, 3)
    _assert_rows(case, {"verify": (ours, _torch_masked(q, kc, vc, qpos), out_r)}, tile=n)
