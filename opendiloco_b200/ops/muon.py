"""Front-ends of the Muon optimizer kernels (``csrc/muon.cu`` and the batched axpby GEMMs of ``csrc/gemm_sm90.cu``) with the
PyTorch reference of each op beside it.

Rounding points (the same in the kernels and the references): momentum, ``u`` and the Frobenius norm in fp32; the
Newton-Schulz iterate X and the products A = X X^T, B = b A + c A A in bf16; every GEMM accumulates in fp32 and rounds
once, after its ``alpha * acc + beta * D`` epilogue.  torch's own ``_zeropower_via_newtonschulz`` normalises in bf16
instead, so results agree with it to about 1e-2 relative, not bit for bit.
"""
from __future__ import annotations

import ctypes as _ct

import torch

from .. import _lib
from .kernels import HP_B1, HP_B2, HP_BC1, HP_BC2, HP_EPS, HP_INVSCALE, HP_LR, HP_MAXNORM, HP_WD  # noqa: F401

BF16 = torch.bfloat16
# hp slots of the Muon group, after the AdamW ones shared with adamw_step (ops/kernels.py)
HP_MLR, HP_MOM, HP_MWD, HP_NESTEROV = 9, 10, 11, 12
TABLE_COLS = 8        # matrix table row: flat offset, rows, cols, transposed, chunk0, chunk1, scratch offset, adjust (f32 bits)

_v, _i, _f, _ll = _ct.c_void_p, _ct.c_int, _ct.c_float, _ct.c_longlong
for _n in ("odb_gemm_batched_axpby_tn", "odb_gemm_batched_axpby_nn"):
    _lib.register_optional(_n, [_v, _v, _v, _v, _i, _i, _i, _i, _ll, _f, _f, _v])
_lib.register_optional("odb_muon_prepare", [_v, _v, _v, _i, _v, _v, _i, _v, _v, _v, _v])
_lib.register_optional("odb_muon_scale", [_v, _i, _v, _v, _i, _v, _v, _f, _v])
_lib.register_optional("odb_muon_normalize", [_v, _v, _v, _i, _i, _i, _v, _v, _v, _v])
_lib.register_optional("odb_muon_apply", [_v, _v, _v, _v, _i, _i, _i, _v, _v, _v, _i, _v])
_lib.register_optional("odb_adamw_segments", [_v, _v, _v, _v, _v, _v, _i, _v, _v, _i, _v, _v, _i, _v])


def _p(t: torch.Tensor | None) -> int | None:
    return None if t is None else t.data_ptr()


def kernel_shape(rows: int, cols: int) -> bool:
    """Matrices the kernels cover; others run ``muon_update_ref`` on their own device."""
    return rows % 64 == 0 and cols % 64 == 0


# ------------------------------------------------------------------------------------------------ batched axpby GEMM
def gemm_batched_axpby(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor, d: torch.Tensor | None, alpha: float, beta: float,
                       b_mn: bool) -> torch.Tensor:
    """c[i] = bf16(alpha * a[i] @ op(b[i]) + beta * d[i]) for bf16 [batch, M, K] a; op(b) = b[i]^T for b [batch, N, K]
    (``b_mn=False``) or b[i] for b [batch, K, N] (``b_mn=True``).  d may be a or b, never c.  M, N, K % 64 == 0 on CUDA."""
    nb, M, K = a.shape
    N = b.shape[2] if b_mn else b.shape[1]
    if a.is_cuda:
        for t in (a, b, c, d):
            assert t is None or (t.dtype == BF16 and t.is_contiguous())
        fn = _lib.cuda_lib().odb_gemm_batched_axpby_nn if b_mn else _lib.cuda_lib().odb_gemm_batched_axpby_tn
        _lib.check(fn(_p(a), _p(b), _p(c), _p(d), nb, M, N, K, N, float(alpha), float(beta), _lib.stream_ptr(a)),
                   "gemm_batched_axpby")
        _lib.count_launch()
        return c
    acc = torch.bmm(a.float(), b.float() if b_mn else b.float().transpose(1, 2)) * alpha
    if d is not None:
        acc = acc + beta * d.float()
    c.copy_(acc.to(c.dtype))
    return c


def newton_schulz(x: torch.Tensor, coeffs: tuple[float, float, float], steps: int, x2: torch.Tensor, amat: torch.Tensor,
                  bmat: torch.Tensor) -> torch.Tensor:
    """``steps`` quintic Newton-Schulz iterations on the stacked bf16 [batch, m, n] x (m <= n, already normalised):
    A = X X^T ; B = b A + c A A ; X = a X + B X.  x2 is a second [batch, m, n] buffer, amat / bmat [batch, m, m].
    Returns whichever of x / x2 holds the result."""
    a, b, c = coeffs
    for _ in range(steps):
        gemm_batched_axpby(x, x, amat, None, 1.0, 0.0, b_mn=False)
        gemm_batched_axpby(amat, amat, bmat, amat, c, b, b_mn=False)      # A symmetric: A A^T = A A
        gemm_batched_axpby(bmat, x, x2, x, 1.0, a, b_mn=True)
        x, x2 = x2, x
    return x


# ------------------------------------------------------------------------------------------------ optimizer step pieces
def clip_coef_ref(hp: torch.Tensor, partials: torch.Tensor, n_partials: int, stats: torch.Tensor | None = None) -> float:
    """The clip coefficient adamw_step applies (1/loss-scale folded in)."""
    inv_scale, max_norm = float(hp[HP_INVSCALE]), float(hp[HP_MAXNORM])
    gnorm = float(partials[:n_partials].double().sum().sqrt()) * inv_scale
    clip = min(1.0, max_norm / (gnorm + 1e-6)) if max_norm > 0 else 1.0
    if stats is not None:
        stats[0], stats[1] = gnorm, clip
    return inv_scale * clip


def muon_update_ref(theta: torch.Tensor, grad: torch.Tensor, buf: torch.Tensor, shadow: torch.Tensor | None, coef: float,
                    lr: float, wd: float, momentum: float, nesterov: bool, coeffs: tuple[float, float, float], steps: int,
                    eps: float, adjust: float, skip: bool) -> None:
    """One Muon update of a single matrix with the kernels' rounding points, on the tensors' own device."""
    if skip:
        return
    gr = grad.float() * coef
    buf.add_((gr - buf) * (1.0 - momentum))
    u = gr + momentum * (buf - gr) if nesterov else buf.clone()
    tall = u.shape[0] > u.shape[1]
    if tall:
        u = u.T
    x = (u / u.norm().clamp(min=eps)).to(BF16)
    a, b, c = coeffs
    for _ in range(steps):
        am = (x.float() @ x.float().T).to(BF16)
        bm = (c * (am.float() @ am.float()) + b * am.float()).to(BF16)
        x = (bm.float() @ x.float() + a * x.float()).to(BF16)
    o = x.float().T if tall else x.float()
    theta.mul_(1.0 - lr * wd).add_(o, alpha=-lr * adjust)
    if shadow is not None:
        shadow.copy_(theta)


def muon_prepare(g: torch.Tensor, buf: torch.Tensor, chunks: torch.Tensor, hp: torch.Tensor, gpart: torch.Tensor, n_gpart: int,
                 found_inf: torch.Tensor | None, upart: torch.Tensor, stats: torch.Tensor | None) -> None:
    """CUDA: clip + momentum update of every chunk (int64 [n, 2] = flat offset, length) and one sum of u^2 per chunk."""
    _lib.check(_lib.cuda_lib().odb_muon_prepare(_p(g), _p(buf), _p(chunks), chunks.shape[0], _p(hp), _p(gpart), n_gpart,
                                                _p(found_inf), _p(upart), _p(stats), _lib.stream_ptr(g)), "muon_prepare")
    _lib.count_launch()


def muon_scale(mats: torch.Tensor, hp: torch.Tensor, gpart: torch.Tensor, n_gpart: int, upart: torch.Tensor,
               scale: torch.Tensor, eps: float) -> None:
    """CUDA: per matrix (chunk range mats[j] = c0, c1): scale[2 c0] = clip coefficient, scale[2 c0 + 1] = 1 / max(||u||, eps)."""
    _lib.check(_lib.cuda_lib().odb_muon_scale(_p(mats), mats.shape[0], _p(hp), _p(gpart), n_gpart, _p(upart), _p(scale),
                                              float(eps), _lib.stream_ptr(hp)), "muon_scale")
    _lib.count_launch()


def muon_normalize(g: torch.Tensor, buf: torch.Tensor, table: torch.Tensor, m: int, n: int, hp: torch.Tensor,
                   scale: torch.Tensor, x: torch.Tensor) -> None:
    """CUDA: x[i] = bf16(u_i * scale) oriented [m, n] for the matrices of ``table`` (int64 [k, 8])."""
    _lib.check(_lib.cuda_lib().odb_muon_normalize(_p(g), _p(buf), _p(table), table.shape[0], m, n, _p(hp), _p(scale), _p(x),
                                                  _lib.stream_ptr(g)), "muon_normalize")
    _lib.count_launch()


def muon_apply(p: torch.Tensor, g: torch.Tensor, shadow: torch.Tensor | None, table: torch.Tensor, m: int, n: int,
               hp: torch.Tensor, x: torch.Tensor, found_inf: torch.Tensor | None, zero_grad: bool) -> None:
    """CUDA: theta = theta (1 - lr wd) - lr adjust O for the matrices of ``table``; bf16 shadow; optional zero-grad."""
    _lib.check(_lib.cuda_lib().odb_muon_apply(_p(p), _p(g), _p(shadow), _p(table), table.shape[0], m, n, _p(hp), _p(x),
                                              _p(found_inf), int(zero_grad), _lib.stream_ptr(p)), "muon_apply")
    _lib.count_launch()


def adamw_segments(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, shadow: torch.Tensor | None,
                   chunks: torch.Tensor, hp: torch.Tensor, gpart: torch.Tensor, n_gpart: int, found_inf: torch.Tensor | None,
                   zero_grad: bool, skipped: torch.Tensor | None = None) -> None:
    """CUDA: adamw_step's update on the chunks (int64 [n, 2] = flat offset, length) of the flat arena, one launch; ``skipped``
    is adamw_step's skipped-step counter."""
    _lib.check(_lib.cuda_lib().odb_adamw_segments(_p(p), _p(g), _p(m), _p(v), _p(shadow), _p(chunks), chunks.shape[0], _p(hp),
                                                  _p(gpart), n_gpart, _p(found_inf), _p(skipped), int(zero_grad),
                                                  _lib.stream_ptr(p)),
               "adamw_segments")
    _lib.count_launch()
