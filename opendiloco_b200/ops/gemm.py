"""GEMM entry points used by the training engine.

Three shapes of GEMM appear in a Llama step (SURVEY.md §2.5 K3/K6/K7):

  * ``mm_nt``      y[M,N]  = a[M,K] @ b[N,K]^T          forward linear        (both operands K-major)
  * ``mm_nn``      y[M,K]  = a[M,N] @ b[N,K]            dgrad                 (b is N-major)
  * ``mm_tn_acc``  w[N,K] += a[T,N]^T @ b[T,K]  (fp32)  wgrad, accumulated straight into the fp32 gradient arena

CUDA bf16 operands always run on the wgmma kernels of ``csrc/gemm_sm90.cu`` (:mod:`opendiloco_b200.ops.tc_gemm`):
``mm_nt`` with K-major operands, ``mm_nn`` with the weight read as an MN-major B operand (no transposed copy),
``mm_tn_acc`` with both operands MN-major and an fp32 reduce-add epilogue.
``torch.mm`` (cuBLAS / ATen) is only the fp32 / fp16 / CPU path and the ``ODB_TC_GEMM=0`` comparison baseline.
"""
from __future__ import annotations

import torch

from . import tc_gemm as TC

_ADDMM_DTYPE_OK: bool | None = None


def mm_nt(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """a[M,K] @ b[N,K]^T : our wgmma kernel for CUDA bf16 operands, cuBLAS/ATen otherwise (fp32, fp16, CPU)."""
    if TC.usable(a, b) and (out is None or TC.usable(out)):
        return TC.linear(a, b, out)
    if out is None:
        return torch.mm(a, b.t())
    return torch.mm(a, b.t(), out=out)


def mm_nn(a: torch.Tensor, b: torch.Tensor, out: torch.Tensor | None = None) -> torch.Tensor:
    """a[M,N] @ b[N,K] (dgrad): the weight ``b`` stays in its forward [out, in] layout and is fed to wgmma as an
    MN-major operand (shared-memory descriptor LBO/SBO), so no transposed weight copy exists."""
    if TC.nn_usable(a, b, out):
        return TC.linear_nn(a, b, out)
    if out is None:
        return torch.mm(a, b)
    return torch.mm(a, b, out=out)


def mm_tn_acc(a: torch.Tensor, b: torch.Tensor, acc: torch.Tensor, alpha: float = 1.0) -> None:
    """acc (fp32 [N,K]) += alpha * a^T @ b with low-precision a [T,N], b [T,K] and fp32 accumulation/output."""
    global _ADDMM_DTYPE_OK
    if (alpha == 1.0 and acc.dtype == torch.float32 and acc.stride(-1) == 1 and acc.data_ptr() % 16 == 0
            and TC.wgrad_usable(a, b)):
        TC.wgrad_acc(a, b, acc)          # wgmma, MN-major operands, split-K, fp32 reduce-add into the grad arena
        return
    if a.dtype == acc.dtype:
        acc.addmm_(a.t(), b, alpha=alpha)
        return
    if a.is_cuda:
        if _ADDMM_DTYPE_OK is None:
            try:
                probe = torch.zeros(8, 8, device=a.device, dtype=torch.float32)
                x = torch.ones(8, 8, device=a.device, dtype=a.dtype)
                torch.addmm(probe, x.t(), x, out_dtype=torch.float32, out=probe)
                _ADDMM_DTYPE_OK = bool(abs(float(probe[0, 0]) - 8.0) < 1e-3)
            except Exception:
                _ADDMM_DTYPE_OK = False
        if _ADDMM_DTYPE_OK:
            torch.addmm(acc, a.t(), b, out_dtype=torch.float32, alpha=alpha, out=acc)
            return
        tmp = torch.mm(a.t(), b, out_dtype=torch.float32)
        acc.add_(tmp, alpha=alpha)
        return
    acc.add_(a.float().t() @ b.float(), alpha=alpha)
