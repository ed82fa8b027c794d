"""FP8 weight-only projections (``generate(fp8_weights=True)``, ``score(fp8_weights=True)``): per-output-row e4m3
quantisation of the decoder-layer projection weights (``csrc/fp8.cu``) and the skinny-M GEMM that streams them at decode
shapes (``csrc/fp8w_gemm_sm90.cu``).

The rule is the per-tensor rule of :mod:`opendiloco_b200.ops.fp8` applied to every row r of a weight W[N, K]:

  amax_r = max |W[r, :]|
  s_r    = 2^floor(log2(448 / amax_r))                 (1 when amax_r = 0; exponent clamped to [-126, 126])
  q[r]   = satfinite_e4m3(W[r, :] * s_r)               (a non-finite amax_r gives NaN bytes and inv_r = NaN)
  inv_r  = 1 / s_r

s_r is a power of two, so the dequantised weight Ŵ = q * inv is a bf16 number and the FP8 GEMM equals the bf16 GEMM on Ŵ
up to accumulation order.  CUDA bf16 tensors run the kernels; everything else runs the references below.
"""
from __future__ import annotations

import ctypes

import torch

from .. import _lib
from .fp8 import _FLT_MAX, _NAN_BYTE, E4M3, FP8_MAX

c_void_p, c_int, c_ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
_lib.register_optional("odb_fp8_quantize_rows", [c_void_p, c_int, c_int, c_void_p])
_lib.register_optional("odb_fp8w_gemm", [c_void_p, c_ll, c_void_p, c_void_p, c_void_p, c_ll, c_void_p, c_int, c_int, c_int, c_int,
                                        c_void_p, c_void_p, c_void_p])

MAX_M = 64                          # tokens per skinny GEMM call; larger M runs the bf16 GEMM on Ŵ
TILE_N = 64                         # weight rows per CTA
SPLIT_UNIT = 256                    # k per split at least (a 64-wide chunk for each of a CTA's four warps)


# ------------------------------------------------------------------------------------------------ references
def row_scale_ref(amax: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(scale, inv, finite) of a vector of fp32 row amaxes: ``ops.fp8.scale_ref`` elementwise."""
    a = amax.float()
    finite = a <= _FLT_MAX
    r = FP8_MAX[E4M3] / a
    e = torch.where(torch.isinf(r), torch.full_like(r, 126), (torch.frexp(r).exponent - 1).float()).clamp(-126, 126)
    scale = torch.where(finite & (a > 0), torch.ldexp(torch.ones_like(r), e), torch.ones_like(r))
    inv = torch.where(finite, 1.0 / scale, torch.full_like(r, float("nan")))
    return scale, inv, finite


def quantize_rows_ref(w: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """(q e4m3 [N, K], inv fp32 [N]) of a weight matrix, one scale per row.  torch turns an e4m3 overflow into NaN instead
    of saturating, so the scaled values are clamped to +-448 first."""
    amax = w.float().abs().amax(dim=1)                                 # NaN propagates
    scale, inv, finite = row_scale_ref(amax)
    m = FP8_MAX[E4M3]
    q = (w.float() * scale[:, None]).clamp(-m, m).to(E4M3)
    q = torch.where(finite[:, None], q.view(torch.uint8), torch.full_like(q.view(torch.uint8), _NAN_BYTE)).view(E4M3)
    return q, inv


def dequantize_rows(q: torch.Tensor, inv: torch.Tensor, dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """Ŵ = q * inv[:, None] in ``dtype`` (exact in bf16 and fp32)."""
    return (q.float() * inv.float()[:, None]).to(dtype)


# ------------------------------------------------------------------------------------------------ quantiser
def quantize_rows(segs: torch.Tensor, n_seg: int, max_rows: int, like: torch.Tensor) -> None:
    """One launch over a device table of bf16 matrices (int64 [n_seg, 6]: src, q, inv, deq pointers, rows, cols): q, inv
    and Ŵ of every row."""
    assert segs.dtype == torch.int64 and segs.is_cuda and segs.is_contiguous()
    _lib.check(_lib.cuda_lib().odb_fp8_quantize_rows(segs.data_ptr(), n_seg, max_rows, _lib.stream_ptr(like)), "fp8_quantize_rows")
    _lib.count_launch()


def quantize_rows_usable(w: torch.Tensor) -> bool:
    return w.is_cuda and w.dtype == torch.bfloat16 and w.is_contiguous() and w.shape[1] % 8 == 0 and w.data_ptr() % 16 == 0


# ------------------------------------------------------------------------------------------------ skinny GEMM
def gemm_shape_ok(N: int, K: int, swiglu: bool = False) -> bool:
    """The skinny GEMM's shapes: K % 128 == 0, N % 64 == 0 (SwiGLU: N = 2I with I % 32 == 0)."""
    return K % 128 == 0 and K >= SPLIT_UNIT and N % TILE_N == 0 and (not swiglu or (N // 2) % (TILE_N // 2) == 0)


def default_splits(N: int, K: int, sms: int) -> int:
    """Split-K factor: enough CTAs for two per SM, at least 256 k per split."""
    tiles = N // TILE_N
    return max(1, min(-(-2 * sms // tiles), K // SPLIT_UNIT))


def workspace_floats(N: int, splits: int) -> int:
    return splits * N * MAX_M if splits > 1 else 0


def linear(x: torch.Tensor, q: torch.Tensor, inv: torch.Tensor, out: torch.Tensor, splits: int = 1,
           ws: torch.Tensor | None = None, counters: torch.Tensor | None = None, act: torch.Tensor | None = None) -> torch.Tensor:
    """out[M, N] = x[M, K] @ (q * inv[:, None])^T, M <= 64, on the skinny kernel.  ``act`` [M, N/2] selects the SwiGLU
    epilogue: out = gate|up and act = silu(gate) * up as ``tc_gemm.linear_swiglu``.  ``splits`` > 1 needs ``ws`` (fp32,
    ``workspace_floats``) and ``counters`` (int32 [N / 64], zero)."""
    M, K = x.shape
    N = q.shape[0]
    assert x.is_cuda and x.dtype == torch.bfloat16 and x.stride(1) == 1 and q.dtype == E4M3 and q.is_contiguous()
    assert inv.dtype == torch.float32 and out.dtype == torch.bfloat16 and out.stride(1) == 1 and 1 <= M <= MAX_M
    if act is not None:
        assert act.is_contiguous() and tuple(act.shape) == (M, N // 2)
    if splits > 1:
        assert ws is not None and ws.numel() >= workspace_floats(N, splits) and counters is not None
        assert counters.dtype == torch.int32 and counters.numel() >= N // TILE_N
    ptr = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
    _lib.check(_lib.cuda_lib().odb_fp8w_gemm(x.data_ptr(), x.stride(0), q.data_ptr(), inv.data_ptr(), out.data_ptr(), out.stride(0),
                                             ptr(act), M, N, K, splits, ptr(ws) if splits > 1 else None,
                                             ptr(counters) if splits > 1 else None, _lib.stream_ptr(x)), "fp8w_gemm")
    _lib.count_launch()
    return out
