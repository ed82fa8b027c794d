"""wgmma GEMM family (fused SwiGLU / RoPE epilogues, weight gradient, MN-major operands) against fp32 PyTorch references."""
import pytest
import torch

from opendiloco_b200.ops import kernels as K
from opendiloco_b200.ops import tc_gemm as T

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


@pytest.mark.parametrize("M,N,Kd", [(128, 256, 64), (300, 520, 200), (1000, 136, 72), (4096, 1024, 1024), (20000, 768, 2688),
                                    (256, 128, 128), (513, 264, 136), (2048, 2048, 512), (8192, 2304, 768), (16384, 1024, 256)])
def test_linear_matches_fp32(M, N, Kd):
    torch.manual_seed(0)
    x = torch.randn(M, Kd, device="cuda").to(BF)
    w = (torch.randn(N, Kd, device="cuda") * 0.1).to(BF)
    out = T.linear(x, w)
    ref = x.float() @ w.float().t()
    assert rel(out, ref) < 4e-3
    assert torch.equal(out, torch.mm(x, w.t()))        # same fp32 accumulation + single bf16 rounding as cuBLAS


@pytest.mark.parametrize("M,c0,N", [(600, 256, 320), (1000, 128, 200)])
def test_linear_strided_views(M, c0, N):
    torch.manual_seed(1)
    big = torch.randn(M, 1024, device="cuda").to(BF)
    x = big[:, c0:c0 + 512]                              # row stride 1024, 512 columns
    w = (torch.randn(N, 512, device="cuda") * 0.1).to(BF)
    outbuf = torch.zeros(M, 2 * N, device="cuda", dtype=BF)
    T.linear(x, w, outbuf[:, N:])
    assert rel(outbuf[:, N:], x.float() @ w.float().t()) < 4e-3
    assert torch.count_nonzero(outbuf[:, :N]) == 0       # TMA store clipped to the view


@pytest.mark.parametrize("M,I,Kd", [(256, 128, 64), (777, 384, 192), (20000, 2688, 1024), (300, 192, 136), (1024, 640, 256),
                                    (4096, 1408, 512)])
def test_swiglu_epilogue(M, I, Kd):
    torch.manual_seed(2)
    x = torch.randn(M, Kd, device="cuda").to(BF)
    w = (torch.randn(2 * I, Kd, device="cuda") * 0.1).to(BF)
    gu, act = torch.empty(M, 2 * I, device="cuda", dtype=BF), torch.empty(M, I, device="cuda", dtype=BF)
    T.linear_swiglu(x, w, gu, act)
    gu_ref = torch.mm(x, w.t())
    assert torch.equal(gu, gu_ref)
    g, u = gu_ref[:, :I].float(), gu_ref[:, I:].float()
    assert rel(act, torch.nn.functional.silu(g) * u) < 4e-3


@pytest.mark.parametrize("B,S,Hq,Hkv,Kd", [(2, 128, 4, 4, 256), (3, 256, 8, 2, 512), (16, 1024, 16, 16, 1024), (1, 64, 2, 1, 128),
                                             (5, 200, 6, 3, 320), (4, 512, 12, 4, 768)])
def test_qkv_rope_epilogue(B, S, Hq, Hkv, Kd):
    torch.manual_seed(3)
    M, N = B * S, (Hq + 2 * Hkv) * 64
    x = torch.randn(M, Kd, device="cuda").to(BF)
    w = (torch.randn(N, Kd, device="cuda") * 0.1).to(BF)
    cos, sin = K.rope_tables(S, 64, 10000.0, "cuda")
    ref = torch.mm(x, w.t())
    v_ref = ref[:, (Hq + Hkv) * 64:].clone()
    K.rope_(ref, cos, sin, S, Hq + Hkv, 64)
    out = torch.empty_like(ref)
    T.linear_qkv_rope(x, w, out, cos, sin, S, (Hq + Hkv) * 64)
    assert rel(out, ref) < 1e-3
    assert torch.equal(out[:, (Hq + Hkv) * 64:], v_ref)   # v is not rotated


@pytest.mark.parametrize("Tn,N,Kd", [(512, 256, 256), (1000, 520, 136), (4096, 1024, 2688), (32768, 768, 512)])
def test_wgrad_accumulates_in_fp32(Tn, N, Kd):
    torch.manual_seed(4)
    dy = torch.randn(Tn, N, device="cuda").to(BF)
    x = torch.randn(Tn, Kd, device="cuda").to(BF)
    acc = torch.randn(N, Kd, device="cuda")
    ref = acc.double() + dy.double().t() @ x.double()
    T.wgrad_acc(dy, x, acc)
    assert rel(acc, ref) < 2e-5
    T.wgrad_acc(dy, x, acc)                                  # accumulation across calls (micro-batches)
    assert rel(acc, ref + dy.double().t() @ x.double()) < 2e-5


def test_wgrad_three_sources_and_views():
    torch.manual_seed(5)
    Tn, Kd = 2048, 512
    dq, dk, dv = (torch.randn(Tn, n, device="cuda").to(BF) for n in (512, 256, 256))
    x = torch.randn(Tn, Kd, device="cuda").to(BF)
    big = torch.zeros(1024 + 256, Kd, device="cuda")
    T.wgrad_acc((dq, dk, dv), x, big[:1024])
    ref = torch.cat([dq, dk, dv], 1).double().t() @ x.double()
    assert rel(big[:1024], ref) < 2e-5 and torch.count_nonzero(big[1024:]) == 0


@pytest.mark.parametrize("M,I,Kd", [(4096, 2048, 256), (8192, 1280, 768), (5000, 2304, 192), (4096, 2688, 1024)])
def test_swiglu_backward_epilogue(M, I, Kd):
    """Down-proj dgrad GEMM with the SwiGLU backward as epilogue == the GEMM followed by the stand-alone kernel."""
    torch.manual_seed(0)
    dy = torch.randn(M, Kd, device="cuda").to(BF)
    w_t = (torch.randn(I, Kd, device="cuda") * 0.1).to(BF)              # down_proj.weight^T: [I, hidden]
    gu = torch.randn(M, 2 * I, device="cuda").to(BF)
    w = w_t.t().contiguous()                                             # down_proj.weight as stored: [hidden, I]
    assert T.swiglu_bwd_usable(dy, w, gu)
    dact = T.linear(dy, w_t)
    ref_unfused = K.swiglu_bwd(dact, gu)
    g, u, d = gu[:, :I].float(), gu[:, I:].float(), dy.float() @ w_t.float().t()
    sg = torch.sigmoid(g)
    ref = torch.cat([d * u * sg * (1 + g * (1 - sg)), d * g * sg], dim=1)
    fused = gu.clone()
    T.linear_swiglu_bwd(dy, w, fused)                                    # weight read MN-major in its forward layout
    assert rel(fused, ref) < 6e-3
    assert rel(fused, ref_unfused) < 2e-3                                # same bf16-rounded d(act), fast-math divide differs
    fused_t = gu.clone()
    T.linear_swiglu_bwd_t(dy, w_t, fused_t)                              # K-major B variant: same MMAs, same result
    assert torch.equal(fused, fused_t)


@pytest.mark.parametrize("M,N,Kd", [(128, 256, 64), (300, 520, 200), (1000, 136, 72), (4096, 1024, 1024), (20000, 1024, 2688),
                                    (8192, 1024, 32000)])
def test_linear_nn_mn_major_b(M, N, Kd):
    """dgrad form: out = a @ b with b [K, N] row-major, fed to wgmma as an MN-major operand (no transposed copy)."""
    torch.manual_seed(6)
    a = torch.randn(M, Kd, device="cuda").to(BF)
    b = (torch.randn(Kd, N, device="cuda") * 0.1).to(BF)
    assert T.nn_usable(a, b)
    out = T.linear_nn(a, b)
    assert rel(out, a.float() @ b.float()) < 4e-3
    assert torch.equal(out, torch.mm(a, b))               # same fp32 accumulation + single rounding as cuBLAS


def test_linear_nn_a3_and_views():
    torch.manual_seed(7)
    M, N = 3000, 512
    big = torch.randn(M, 1024, device="cuda").to(BF)
    dq, dk, dv = big[:, :512], big[:, 512:768], big[:, 768:]
    w = (torch.randn(1024, N, device="cuda") * 0.1).to(BF)
    out = torch.empty(M, N, device="cuda", dtype=BF)
    T.linear_nn_a3(dq, dk, dv, w, out)
    assert torch.equal(out, torch.mm(big, w))
