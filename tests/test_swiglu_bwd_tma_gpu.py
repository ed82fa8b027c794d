"""Fused down-projection dgrad + SwiGLU backward (kSwiGLUBwd) with its gate / up inputs carried through the operand ring
and d(gate) | d(up) stored by TMA: the bench shape, partial last m- and n-tiles, tiles with fewer k-blocks than ring
entries, the K-major and MN-major weight operands, the FP8 variant, and back-to-back calls."""
import pytest
import torch

from opendiloco_b200.ops import fp8 as F
from opendiloco_b200.ops import kernels as K
from opendiloco_b200.ops import tc_gemm as T

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


def _inputs(M, I, Kd, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    dy = torch.randn(M, Kd, device="cuda", generator=g).to(BF)
    w_t = (torch.randn(I, Kd, device="cuda", generator=g) * 0.1).to(BF)      # down_proj.weight^T: [I, hidden]
    gu = torch.randn(M, 2 * I, device="cuda", generator=g).to(BF)
    return dy, w_t, gu


def _unfused(dy, w_t, gu):
    """The down-projection dgrad GEMM, then the stand-alone SwiGLU backward kernel."""
    return K.swiglu_bwd(T.linear(dy, w_t), gu)


# (32768, 2688, 1024): the Llama-150M step (21+ tiles per CTA, last n-tile half beyond I); (5000, 2688, 1024): partial last
# m-tile; (4096, 2304, 512): I a multiple of 256; (32768, 1024, 64) and (9000, 768, 192): fewer k-blocks per tile than
# the tile has epilogue ring entries, so the ring's phase runs ahead of the k-block count
@pytest.mark.parametrize("M,I,Kd", [(32768, 2688, 1024), (5000, 2688, 1024), (4096, 2304, 512), (32768, 1024, 64), (9000, 768, 192)])
def test_matches_unfused_and_k_major_variant(M, I, Kd):
    dy, w_t, gu = _inputs(M, I, Kd, seed=M + I + Kd)
    w = w_t.t().contiguous()                                             # down_proj.weight as stored: [hidden, I]
    assert T.swiglu_bwd_usable(dy, w, gu)
    ref = _unfused(dy, w_t, gu)
    fused = gu.clone()
    T.linear_swiglu_bwd(dy, w, fused)
    assert rel(fused, ref) < 2e-3                                        # same bf16 d(act); the sigmoids differ slightly
    fused_t = gu.clone()
    T.linear_swiglu_bwd_t(dy, w_t, fused_t)
    assert torch.equal(fused, fused_t)


def test_rows_past_m_untouched():
    """gu is the first M rows of a larger buffer: the partial last m-tile loads zeros past M and its stores are clipped."""
    M, I, Kd, extra = 5000, 2688, 1024, 200
    dy, w_t, gu = _inputs(M, I, Kd, seed=11)
    big = torch.randn(M + extra, 2 * I, device="cuda").to(BF)
    tail = big[M:].clone()
    big[:M].copy_(gu)
    T.linear_swiglu_bwd(dy, w_t.t().contiguous(), big[:M])
    assert torch.equal(big[M:], tail)
    assert rel(big[:M], _unfused(dy, w_t, gu)) < 2e-3


def test_back_to_back_calls_on_different_buffers():
    M, I, Kd = 8192, 2688, 1024
    dy1, w_t, gu1 = _inputs(M, I, Kd, seed=21)
    dy2, _, gu2 = _inputs(M, I, Kd, seed=22)
    w = w_t.t().contiguous()
    ref1, ref2 = _unfused(dy1, w_t, gu1), _unfused(dy2, w_t, gu2)
    a, b = gu1.clone(), gu2.clone()
    T.linear_swiglu_bwd(dy1, w, a)
    T.linear_swiglu_bwd(dy2, w, b)                                       # no synchronisation in between
    solo = gu2.clone()
    torch.cuda.synchronize()
    T.linear_swiglu_bwd(dy2, w, solo)
    assert torch.equal(b, solo)
    assert rel(a, ref1) < 2e-3 and rel(b, ref2) < 2e-3


@pytest.mark.parametrize("M", [4096, 5000])
def test_fp8_matches_bf16_on_dequantised_operands(M):
    I, Kd = 2688, 1024
    Mq = (M + 63) // 64 * 64                                             # the cast takes whole 64-row blocks
    dy, w_t, _ = _inputs(Mq, I, Kd, seed=31)
    gu = _inputs(M, I, Kd, seed=32)[2]

    def q(x, fmt):
        slot, inv = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
        out = torch.empty(x.shape, dtype=fmt, device="cuda")
        F.quantize(x, slot, inv, fmt, out=out)
        return out, inv

    (dy8, idy), (wdt8, iwd) = q(dy, F.E5M2), q(w_t, F.E4M3)
    dy8 = dy8[:M]                                                        # M = 5000: a partial last m-tile
    g8, g16 = gu.clone(), gu.clone()
    F.linear_swiglu_bwd(dy8, wdt8, idy, iwd, g8)
    T.linear_swiglu_bwd_t(F.dequantize(dy8, idy), F.dequantize(wdt8, iwd), g16)
    assert rel(g8, g16) < 5e-3                                           # FP8 accumulation inside each 128-deep k-block
