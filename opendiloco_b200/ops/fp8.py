"""FP8 (``precision="fp8-mixed"``) ops: per-tensor current scaling and the FP8 wgmma GEMMs (``csrc/fp8.cu``,
``csrc/gemm_sm90.cu``).

The recipe, for every quantised tensor of a micro-step:

  amax  = max |x|                                     (device scalar; inf / NaN propagate)
  scale = 2^floor(log2(FP8_MAX / amax))               (1 when amax = 0; FP8_MAX = 448 for e4m3, 57344 for e5m2)
  q     = round_to_nearest_even(clamp(x * scale))     (a non-finite amax gives the FP8 NaN byte everywhere)
  inv   = 1 / scale                                   (device scalar read by the GEMM epilogue)

e4m3 holds activations and weights, e5m2 the gradients that flow backward.  Scales are powers of two, so x * scale and
q * inv are exact and an FP8 GEMM equals the bf16 GEMM of the quantised-dequantised ("QDQ") operands up to accumulation
order: every reference below is that bf16 GEMM (:mod:`opendiloco_b200.ops.gemm`, our bf16 kernels on CUDA).

FP8 tensors are torch ``float8_e4m3fn`` / ``float8_e5m2`` tensors.  CUDA tensors run the kernels; CPU tensors run the
reference next to each op, so the CPU test-suite executes the whole FP8 program.
"""
from __future__ import annotations

import ctypes

import torch

from .. import _lib
from . import attention as A
from . import gemm as G
from . import kernels as K

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
FP8_MAX = {E4M3: 448.0, E5M2: 57344.0}
_NAN_BYTE = 0x7F                        # NaN in both e4m3fn and e5m2
_FLT_MAX = torch.finfo(torch.float32).max

c_void_p, c_int, c_ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
_lib.register_optional("odb_fp8_amax", [c_void_p, c_ll, c_void_p, c_void_p])
_lib.register_optional("odb_fp8_cast", [c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p])
_lib.register_optional("odb_gemm_fp8_tn", [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_ll, c_ll, c_int, c_void_p,
                                          c_void_p, c_void_p])
_lib.register_optional("odb_gemm_fp8_qkv_rope", [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                                                c_void_p, c_void_p, c_void_p])
_lib.register_optional("odb_gemm_fp8_swiglu", [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                                              c_void_p])
_lib.register_optional("odb_gemm_fp8_swiglu_bwd", [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_ll, c_void_p, c_void_p,
                                                  c_void_p])
_lib.register_optional("odb_wgrad_fp8", [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_ll, c_ll, c_ll, c_void_p, c_void_p,
                                        c_void_p])


def _p(t: torch.Tensor | None):
    return t.data_ptr() if t is not None else None


# ------------------------------------------------------------------------------------------------ configuration
def check_config(cfg) -> None:
    """Raise ValueError when a model shape falls outside what the CUDA FP8 kernels cover.

    The casts work on 64 x 64 tiles and the FP8 GEMMs on K-major operands whose rows are multiples of 16 bytes; the fused
    QKV + RoPE epilogue needs 64-wide heads.  So: head_dim == 64 and hidden_size, intermediate_size % 64 == 0 (q/k/v
    widths are then multiples of 64 too).  The token count B * S must be a multiple of 64 (checked per batch shape).
    The FP8 weight gradient of the QKV projection takes the packed dq|dk|dv of the project's attention backward, so a
    library attention (``ODB_ATTN_LIB``) is refused."""
    if cfg.head_dim != 64:
        raise ValueError(f"precision='fp8-mixed' needs head_dim == 64 on CUDA (got head_dim={cfg.head_dim})")
    for name in ("hidden_size", "intermediate_size"):
        v = getattr(cfg, name)
        if v % 64:
            raise ValueError(f"precision='fp8-mixed' needs {name} % 64 == 0 on CUDA (got {name}={v})")
    if A._LIB != "tc":
        raise ValueError(f"precision='fp8-mixed' runs on the project's attention kernels only; ODB_ATTN_LIB={A._LIB!r} selects "
                         "a library attention whose un-packed dq/dk/dv the FP8 weight gradient does not take")


def check_tokens(T: int) -> None:
    if T % 64:
        raise ValueError(f"precision='fp8-mixed' needs batch * sequence length % 64 == 0 on CUDA (got {T} tokens)")


# ------------------------------------------------------------------------------------------------ references
def scale_ref(amax: torch.Tensor, fmt: torch.dtype) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """(scale, inv, finite) of a 1-element fp32 amax, exactly as the cast kernel derives them."""
    a = amax.reshape(1).float()
    finite = a <= _FLT_MAX                                         # False for inf and NaN
    r = torch.tensor([FP8_MAX[fmt]], dtype=torch.float32, device=a.device) / a
    e = torch.where(torch.isinf(r), torch.full_like(r, 126), (torch.frexp(r).exponent - 1).float()).clamp(-126, 126)
    scale = torch.where(finite & (a > 0), torch.ldexp(torch.ones_like(r), e), torch.ones_like(r))
    inv = torch.where(finite, 1.0 / scale, torch.full_like(r, float("nan")))
    return scale, inv, finite


def quantize_ref(x: torch.Tensor, fmt: torch.dtype, amax: torch.Tensor | None = None) -> tuple[torch.Tensor, torch.Tensor]:
    """(q, inv): q = FP8 copy of x with the scale of ``amax`` (default: max |x|).  torch turns an e4m3 overflow into NaN
    instead of saturating, so the scaled values are clamped to +-FP8_MAX first."""
    if amax is None:
        amax = x.float().abs().amax().reshape(1)
    scale, inv, finite = scale_ref(amax, fmt)
    m = FP8_MAX[fmt]
    q = (x.float() * scale).clamp(-m, m).to(fmt)
    nan = torch.full_like(q.view(torch.uint8), _NAN_BYTE)
    q = torch.where(finite, q.view(torch.uint8), nan).view(fmt)
    return q, inv


def dequantize(q: torch.Tensor, inv: torch.Tensor) -> torch.Tensor:
    """bf16 value of an FP8 tensor (exact: FP8 values times a power of two are bf16 numbers)."""
    return (q.float() * inv.reshape(1).float()).to(torch.bfloat16)


def qdq(x: torch.Tensor, fmt: torch.dtype) -> torch.Tensor:
    """Quantise-dequantise: the bf16 tensor an FP8 GEMM effectively multiplies."""
    return dequantize(*quantize_ref(x, fmt))


# ------------------------------------------------------------------------------------------------ casts
def amax(x: torch.Tensor, slot: torch.Tensor) -> None:
    """slot (fp32, 1 element) = max |x|.  The slot is reset in-stream: CUDA-graph capturable."""
    if x.is_cuda:
        assert x.dtype == torch.bfloat16 and x.is_contiguous() and slot.dtype == torch.float32
        _lib.check(_lib.cuda_lib().odb_fp8_amax(_p(x), x.numel(), _p(slot), _lib.stream_ptr(x)), "fp8_amax")
        _lib.count_launch()
    else:
        slot.copy_(x.float().abs().amax().reshape(1))


def cast(x: torch.Tensor, slot: torch.Tensor, fmt: torch.dtype, inv: torch.Tensor, out: torch.Tensor | None = None,
         out_t: torch.Tensor | None = None) -> None:
    """FP8 copies of x [R, C] with the scale derived from ``slot``: ``out`` [R, C] and / or ``out_t`` [C, R] (the transposed
    copy, the K-major operand of the weight gradient); ``inv`` (fp32, 1 element) = 1 / scale."""
    assert out is not None or out_t is not None
    if x.is_cuda:
        R, C = x.shape
        assert x.dtype == torch.bfloat16 and x.is_contiguous()
        for t in (out, out_t):
            assert t is None or (t.dtype == fmt and t.is_contiguous())
        _lib.check(_lib.cuda_lib().odb_fp8_cast(_p(x), R, C, _p(slot), int(fmt == E5M2), _p(out), _p(out_t), _p(inv),
                                                _lib.stream_ptr(x)), "fp8_cast")
        _lib.count_launch()
        return
    q, iv = quantize_ref(x, fmt, slot)
    if out is not None:
        out.copy_(q)
    if out_t is not None:
        out_t.copy_(q.t())
    inv.copy_(iv)


def quantize(x: torch.Tensor, slot: torch.Tensor, inv: torch.Tensor, fmt: torch.dtype, out: torch.Tensor | None = None,
             out_t: torch.Tensor | None = None) -> None:
    """amax into ``slot``, then ``cast``."""
    amax(x, slot)
    cast(x, slot, fmt, inv, out, out_t)


# ------------------------------------------------------------------------------------------------ GEMMs
def linear(a: torch.Tensor, b: torch.Tensor, inv_a: torch.Tensor, inv_b: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out[M, N] (bf16) = a[M, K] @ b[N, K]^T * inv_a * inv_b: forward projections (a e4m3) and dgrads (a e5m2, b the
    transposed weight)."""
    M, Kd = a.shape
    N = b.shape[0]
    if a.is_cuda:
        assert b.dtype == E4M3 and a.dtype in (E4M3, E5M2) and out.stride(1) == 1
        _lib.check(_lib.cuda_lib().odb_gemm_fp8_tn(_p(a), _p(b), _p(out), M, N, Kd, a.stride(0), b.stride(0), out.stride(0),
                                                   int(a.dtype == E5M2), _p(inv_a), _p(inv_b), _lib.stream_ptr(a)), "gemm_fp8_tn")
        _lib.count_launch()
        return out
    return G.mm_nt(dequantize(a, inv_a), dequantize(b, inv_b), out=out)


def linear_qkv_rope(x: torch.Tensor, w: torch.Tensor, inv_x: torch.Tensor, inv_w: torch.Tensor, qkv: torch.Tensor,
                    cos: torch.Tensor, sin: torch.Tensor, S: int, n_rot_heads: int, D: int) -> None:
    """qkv = x @ w^T with RoPE on the first n_rot_heads heads (q | k), as ``tc_gemm.linear_qkv_rope``."""
    M, Kd = x.shape
    N = w.shape[0]
    if x.is_cuda:
        assert D == 64 and x.dtype == E4M3 and w.dtype == E4M3 and qkv.is_contiguous()
        _lib.check(_lib.cuda_lib().odb_gemm_fp8_qkv_rope(_p(x), _p(w), _p(qkv), M, N, Kd, S, n_rot_heads * D, _p(cos), _p(sin),
                                                         _p(inv_x), _p(inv_w), _lib.stream_ptr(x)), "gemm_fp8_qkv_rope")
        _lib.count_launch()
        return
    G.mm_nt(dequantize(x, inv_x), dequantize(w, inv_w), out=qkv)
    K.rope_(qkv, cos, sin, S, n_rot_heads, D)


def linear_swiglu(x: torch.Tensor, w_gu: torch.Tensor, inv_x: torch.Tensor, inv_w: torch.Tensor, gu: torch.Tensor,
                  act: torch.Tensor) -> None:
    """gu = x @ w_gu^T and act = silu(gate) * up, as ``tc_gemm.linear_swiglu``."""
    M, Kd = x.shape
    I = w_gu.shape[0] // 2
    if x.is_cuda:
        assert x.dtype == E4M3 and w_gu.dtype == E4M3 and gu.is_contiguous() and act.is_contiguous()
        _lib.check(_lib.cuda_lib().odb_gemm_fp8_swiglu(_p(x), _p(w_gu), _p(gu), _p(act), M, I, Kd, _p(inv_x), _p(inv_w),
                                                       _lib.stream_ptr(x)), "gemm_fp8_swiglu")
        _lib.count_launch()
        return
    G.mm_nt(dequantize(x, inv_x), dequantize(w_gu, inv_w), out=gu)
    K.swiglu_fwd(gu, out=act)


def linear_swiglu_bwd(dy: torch.Tensor, w_down_t: torch.Tensor, inv_dy: torch.Tensor, inv_w: torch.Tensor, gu: torch.Tensor) -> None:
    """gu [M, 2I] (gate|up) <- d(gate)|d(up) in place, d(act) = dy @ w_down_t^T formed in registers only
    (e5m2 dy [M, h], e4m3 w_down_t [I, h] = the transposed down-projection weight)."""
    M, Kd = dy.shape
    I = w_down_t.shape[0]
    if dy.is_cuda:
        assert dy.dtype == E5M2 and w_down_t.dtype == E4M3 and gu.is_contiguous() and gu.shape[1] == 2 * I
        _lib.check(_lib.cuda_lib().odb_gemm_fp8_swiglu_bwd(_p(dy), _p(w_down_t), _p(gu), M, I, Kd, dy.stride(0), w_down_t.stride(0),
                                                           _p(inv_dy), _p(inv_w), _lib.stream_ptr(dy)), "gemm_fp8_swiglu_bwd")
        _lib.count_launch()
        return
    dact = G.mm_nt(dequantize(dy, inv_dy), dequantize(w_down_t, inv_w))
    K.swiglu_bwd(dact, gu, gu)


def wgrad(dy_t: torch.Tensor, x_t: torch.Tensor, inv_dy: torch.Tensor, inv_x: torch.Tensor, dw: torch.Tensor) -> None:
    """dw (fp32 [N_out, K_out]) += dy_t[N_out, T] @ x_t[K_out, T]^T: the weight gradient on the transposed copies
    (e5m2 gradient, e4m3 activation), split-K over tokens with an fp32 reduce-add."""
    N_out, T = dy_t.shape
    K_out = x_t.shape[0]
    assert dw.dtype == torch.float32 and dw.stride(1) == 1 and tuple(dw.shape) == (N_out, K_out)
    if dy_t.is_cuda:
        assert dy_t.dtype == E5M2 and x_t.dtype == E4M3
        _lib.check(_lib.cuda_lib().odb_wgrad_fp8(_p(dy_t), _p(x_t), _p(dw), N_out, K_out, T, dy_t.stride(0), x_t.stride(0),
                                                 dw.stride(0), _p(inv_dy), _p(inv_x), _lib.stream_ptr(dy_t)), "wgrad_fp8")
        _lib.count_launch()
        return
    G.mm_tn_acc(dequantize(dy_t, inv_dy).t(), dequantize(x_t, inv_x).t(), dw)
