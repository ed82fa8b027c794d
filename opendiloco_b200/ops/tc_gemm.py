"""Python front-end of the wgmma GEMM family (``csrc/gemm_sm90.cu``).

``linear``         y = x @ W^T                                  (bf16 in/out, fp32 accumulate)
``linear_swiglu``  gu = x @ Wgu^T ; act = silu(gate) * up        (one kernel: the SwiGLU pass is the GEMM epilogue)
``linear_qkv_rope`` qkv = x @ Wqkv^T with RoPE on the q|k heads   (RoPE is the GEMM epilogue; head_dim 64)

All three require CUDA bf16 tensors with contiguous rows; callers fall back to the library GEMM + stand-alone kernels
for other dtypes/devices (CPU tests, fp32 runs)."""
from __future__ import annotations

import ctypes
import os

import torch

from .. import _lib

c_void_p, c_int, c_ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
_lib.register_optional("odb_gemm_bf16_tn", [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_ll, c_ll, c_void_p])
_lib.register_optional("odb_gemm_swiglu", [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p])
_lib.register_optional("odb_gemm_qkv_rope", [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p])

_lib.register_optional("odb_wgrad_bf16", [c_void_p, c_void_p, c_void_p, c_ll, c_ll, c_ll, c_int, c_int, c_int, c_void_p, c_ll, c_void_p,
                                         c_ll, c_int, c_int, c_void_p])

_lib.register_optional("odb_gemm_swiglu_bwd", [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_ll, c_void_p])

_lib.register_optional("odb_gemm_bf16_nn", [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_ll, c_ll, c_void_p])
_lib.register_optional("odb_gemm_bf16_nn_a3", [c_void_p, c_void_p, c_void_p, c_ll, c_ll, c_ll, c_int, c_int, c_int, c_void_p, c_void_p,
                                               c_int, c_int, c_ll, c_ll, c_void_p])
_lib.register_optional("odb_gemm_swiglu_bwd_nn", [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_ll, c_void_p])
_lib.register_optional("odb_lce_fwd", [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_ll, c_ll, c_void_p, c_void_p, c_int,
                                      c_int, c_void_p])
_lib.register_optional("odb_lce_planes", [c_int])
_lib.register_optional("odb_lce_dx", [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_ll, c_ll, c_void_p, c_void_p, c_void_p,
                                     c_void_p])
_lib.register_optional("odb_lce_score", [c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_ll, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_void_p])
SCORE_PLANE = 256                   # vocabulary columns per plane of the scoring statistics (the GEMM's tile width)

ENABLED = os.environ.get("ODB_TC_GEMM", "1") != "0"


def usable(*tensors: torch.Tensor) -> bool:
    """CUDA bf16 matrices with contiguous rows whose row stride and width are multiples of 8 elements (16-byte TMA rows)
    and whose base is 16-byte aligned (TMA reads the operands and stores the output); anything else (e.g. an odd
    vocabulary size, a view starting at an odd column) takes the library GEMM."""
    return ENABLED and all(t.is_cuda and t.dtype == torch.bfloat16 and t.stride(-1) == 1 and t.data_ptr() % 16 == 0 and
                           (t.dim() < 2 or (t.stride(0) % 8 == 0 and t.shape[-1] % 8 == 0)) for t in tensors)


def linear(x: torch.Tensor, w: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    M, K = x.shape
    N = w.shape[0]
    if out is None:
        out = torch.empty(M, N, dtype=x.dtype, device=x.device)
    _lib.check(_lib.cuda_lib().odb_gemm_bf16_tn(x.data_ptr(), w.data_ptr(), out.data_ptr(), M, N, K, x.stride(0), w.stride(0),
                                                 out.stride(0), _lib.stream_ptr(x)), "gemm_bf16_tn")
    _lib.count_launch()
    return out


def linear_swiglu(x: torch.Tensor, w_gu: torch.Tensor, gu: torch.Tensor, act: torch.Tensor) -> None:
    M, K = x.shape
    I = w_gu.shape[0] // 2
    assert x.is_contiguous() and w_gu.is_contiguous() and gu.is_contiguous() and act.is_contiguous()
    _lib.check(_lib.cuda_lib().odb_gemm_swiglu(x.data_ptr(), w_gu.data_ptr(), gu.data_ptr(), act.data_ptr(), M, I, K,
                                                _lib.stream_ptr(x)), "gemm_swiglu")
    _lib.count_launch()


def swiglu_bwd_usable(dy: torch.Tensor, w_down: torch.Tensor, gu: torch.Tensor) -> bool:
    """The fused down-proj dgrad + SwiGLU backward (``w_down`` is the weight in its forward [h, I] layout)."""
    if not usable(dy, w_down, gu):
        return False
    I = w_down.shape[1]
    return I % 64 == 0 and gu.is_contiguous() and gu.shape[1] == 2 * I


def linear_swiglu_bwd(dy: torch.Tensor, w_down: torch.Tensor, gu: torch.Tensor) -> None:
    """gu [M, 2I] (gate|up) <- d(gate)|d(up) in place, with d(act) = dy @ w_down formed in registers only
    (replaces the down-proj dgrad GEMM + the stand-alone swiglu_bwd kernel: d(act) is neither written nor re-read).
    ``w_down`` [h, I] is read as an MN-major B operand, i.e. exactly as the forward pass stores it."""
    M, K = dy.shape
    I = w_down.shape[1]
    _lib.check(_lib.cuda_lib().odb_gemm_swiglu_bwd_nn(dy.data_ptr(), w_down.data_ptr(), gu.data_ptr(), M, I, K, dy.stride(0),
                                                       w_down.stride(0), _lib.stream_ptr(dy)), "gemm_swiglu_bwd_nn")
    _lib.count_launch()


def linear_swiglu_bwd_t(dy: torch.Tensor, w_down_t: torch.Tensor, gu: torch.Tensor) -> None:
    """Same with the weight given transposed ([I, h], K-major B) - kept for the kernel tests."""
    M, K = dy.shape
    I = w_down_t.shape[0]
    _lib.check(_lib.cuda_lib().odb_gemm_swiglu_bwd(dy.data_ptr(), w_down_t.data_ptr(), gu.data_ptr(), M, I, K, dy.stride(0),
                                                    w_down_t.stride(0), _lib.stream_ptr(dy)), "gemm_swiglu_bwd")
    _lib.count_launch()


def nn_usable(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor | None = None) -> bool:
    return usable(a, b) and (out is None or usable(out)) and b.shape[1] % 8 == 0 and a.shape[1] % 8 == 0


def linear_nn(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """out[M, N] = a[M, K] @ b[K, N] with b row-major (the dgrad dX = dY W on the forward weight layout): B is fed to
    wgmma as an MN-major operand, no transposed weight copy exists anywhere."""
    M, K = a.shape
    N = b.shape[1]
    if out is None:
        out = torch.empty(M, N, dtype=a.dtype, device=a.device)
    _lib.check(_lib.cuda_lib().odb_gemm_bf16_nn(a.data_ptr(), b.data_ptr(), out.data_ptr(), M, N, K, a.stride(0), b.stride(0),
                                                 out.stride(0), _lib.stream_ptr(a)), "gemm_bf16_nn")
    _lib.count_launch()
    return out


def linear_nn_a3(a0: torch.Tensor, a1: torch.Tensor, a2: torch.Tensor, w: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out = cat([a0, a1, a2], dim=1) @ w with w [K0+K1+K2, N] row-major; the three A pieces are read in place."""
    M = a0.shape[0]
    N = w.shape[1]
    _lib.check(_lib.cuda_lib().odb_gemm_bf16_nn_a3(a0.data_ptr(), a1.data_ptr(), a2.data_ptr(), a0.stride(0), a1.stride(0),
                                                    a2.stride(0), a0.shape[1], a1.shape[1], a2.shape[1], w.data_ptr(), out.data_ptr(),
                                                    M, N, w.stride(0), out.stride(0), _lib.stream_ptr(out)), "gemm_bf16_nn_a3")
    _lib.count_launch()
    return out


# ------------------------------------------------------------------------------------------------ fused linear-cross-entropy
def lce_usable(x: torch.Tensor, w: torch.Tensor) -> bool:
    return usable(x, w) and w.shape[1] % 64 == 0 and w.shape[0] % 8 == 0


def lce_planes(V: int) -> int:
    return int(_lib.cuda_lib().odb_lce_planes(V))


def lce_fwd(x: torch.Tensor, w: torch.Tensor, shift: torch.Tensor, partials: torch.Tensor, e_out: torch.Tensor | None,
            want_sumsq: bool = False) -> None:
    """LM-head GEMM whose epilogue emits e = exp(x @ w^T - shift[:, None]) (bf16, only when ``e_out`` is given) and the
    partial row sums of e (``partials`` [planes(, x2 with want_sumsq), M] fp32; one plane per 256 vocabulary columns).  Logits are never written."""
    M, K = x.shape
    V = w.shape[0]
    assert partials.dtype == torch.float32 and partials.numel() >= lce_planes(V) * M * (2 if want_sumsq else 1)
    _lib.check(_lib.cuda_lib().odb_lce_fwd(x.data_ptr(), w.data_ptr(), e_out.data_ptr() if e_out is not None else None, M, V, K,
                                           x.stride(0), w.stride(0), e_out.stride(0) if e_out is not None else 0,
                                           shift.data_ptr(), partials.data_ptr(), int(want_sumsq), int(e_out is not None),
                                           _lib.stream_ptr(x)), "lce_fwd")
    _lib.count_launch()


def lce_dx(e: torch.Tensor, w: torch.Tensor, rowscale: torch.Tensor, labels: torch.Tensor, gscale: torch.Tensor,
           out: torch.Tensor) -> None:
    """out[M, h] = rowscale[:, None] * (e @ w) - gscale * w[labels]   (rows with label < 0 get rowscale 0 and no gather)."""
    M, V = e.shape
    N = w.shape[1]
    _lib.check(_lib.cuda_lib().odb_lce_dx(e.data_ptr(), w.data_ptr(), out.data_ptr(), M, N, V, e.stride(0), w.stride(0),
                                          out.stride(0), rowscale.data_ptr(), labels.data_ptr(), gscale.data_ptr(),
                                          _lib.stream_ptr(e)), "lce_dx")
    _lib.count_launch()


def lce_score(x: torch.Tensor, w: torch.Tensor, labels: torch.Tensor, pmax: torch.Tensor, psum: torch.Tensor, pidx: torch.Tensor,
              zlab: torch.Tensor) -> None:
    """Scoring statistics of the logits z = x @ w^T without writing them.  Per row and plane of 256 vocabulary columns
    (``planes = ceil(V / 256)``; the flat buffers hold [planes, M] with row stride M): ``pmax`` = the plane maximum,
    ``pidx`` (int32) = its lowest column, ``psum`` = sum exp(z - pmax); ``zlab[:M]`` = z[label] (untouched where label < 0).

    CUDA bf16: the kLCEScore epilogue of the wgmma GEMM.  Other dtypes / CPU: the reference on the fp32 logits chunk."""
    M = x.shape[0]
    V = w.shape[0]
    planes = (V + SCORE_PLANE - 1) // SCORE_PLANE
    assert pmax.numel() >= planes * M and psum.numel() >= planes * M and pidx.numel() >= planes * M and zlab.numel() >= M
    assert pidx.dtype == torch.int32 and labels.dtype == torch.int64 and labels.is_contiguous()
    if lce_usable(x, w):
        _lib.check(_lib.cuda_lib().odb_lce_score(x.data_ptr(), w.data_ptr(), M, V, x.shape[1], x.stride(0), w.stride(0), labels.data_ptr(),
                                                 pmax.data_ptr(), psum.data_ptr(), pidx.data_ptr(), zlab.data_ptr(), _lib.stream_ptr(x)),
                   "lce_score")
        _lib.count_launch()
        return
    z = x.float() @ w.float().t()                                                  # [M, V] fp32 logits chunk
    zp = torch.nn.functional.pad(z, (0, planes * SCORE_PLANE - V), value=float("-inf")).view(M, planes, SCORE_PLANE)
    m = zp.amax(dim=-1)
    pmax[: planes * M].view(planes, M).copy_(m.t())
    psum[: planes * M].view(planes, M).copy_(torch.exp(zp - m[..., None]).sum(dim=-1).t())
    first = torch.arange(planes, device=z.device, dtype=torch.int64) * SCORE_PLANE
    pidx[: planes * M].view(planes, M).copy_((zp.argmax(dim=-1) + first).t())     # argmax: the first maximal index
    valid = labels >= 0
    zl = z.gather(1, labels.clamp(min=0)[:, None])[:, 0]
    zlab[:M].copy_(torch.where(valid, zl, zlab[:M]))


def linear_qkv_rope(x: torch.Tensor, w: torch.Tensor, qkv: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, S: int,
                    rope_cols: int) -> None:
    M, K = x.shape
    N = w.shape[0]
    assert x.is_contiguous() and w.is_contiguous() and qkv.is_contiguous() and cos.shape[1] == 32
    _lib.check(_lib.cuda_lib().odb_gemm_qkv_rope(x.data_ptr(), w.data_ptr(), qkv.data_ptr(), M, N, K, S, rope_cols, cos.data_ptr(),
                                                  sin.data_ptr(), _lib.stream_ptr(x)), "gemm_qkv_rope")
    _lib.count_launch()


def wgrad_usable(*tensors: torch.Tensor) -> bool:
    return usable(*tensors)


def wgrad_acc(dy, x: torch.Tensor, dw: torch.Tensor) -> None:
    """dw (fp32 [N_out, K_out]) += dy^T @ x, reduction over tokens.  ``dy`` is one [T, N_out] matrix or a tuple of up to
    three matrices whose columns are concatenated (dq | dk | dv; every piece a multiple of 256 columns)."""
    parts = list(dy) if isinstance(dy, (tuple, list)) else [dy]
    assert 1 <= len(parts) <= 3 and dw.dtype == torch.float32 and dw.stride(1) == 1
    T, K_out = x.shape
    while len(parts) < 3:
        parts.append(None)
    ptr = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
    ld = lambda t: t.stride(0) if t is not None else 0        # noqa: E731
    nc = lambda t: t.shape[1] if t is not None else 0         # noqa: E731
    _lib.check(_lib.cuda_lib().odb_wgrad_bf16(ptr(parts[0]), ptr(parts[1]), ptr(parts[2]), ld(parts[0]), ld(parts[1]), ld(parts[2]),
                                              nc(parts[0]), nc(parts[1]), nc(parts[2]), x.data_ptr(), x.stride(0), dw.data_ptr(),
                                              dw.stride(0), T, K_out, _lib.stream_ptr(x)), "wgrad_bf16")
    _lib.count_launch()
