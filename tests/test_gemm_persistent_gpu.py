"""Persistent wgmma GEMMs with TMA-stored epilogues: many tiles per CTA (the stage ring wraps across tiles), partial edge
tiles clipped by the output tensor map, split-K items outnumbering the grid, a store still in flight when the next
kernel reads, and outputs the TMA cannot store (misaligned) falling back."""
import pytest
import torch

from opendiloco_b200.ops import gemm as G
from opendiloco_b200.ops import kernels as K
from opendiloco_b200.ops import tc_gemm as T

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


# 32768 x 1024 is 1024 tiles (7.8 per CTA on 132 SMs); 33000 x 1000 has partial tiles in M and N; 256 x 512 has 4 tiles
SHAPES = [(32768, 1024, 1024), (32768, 3072, 1024), (32768, 1024, 3072), (33000, 1000, 1032), (256, 512, 256)]


@pytest.mark.parametrize("M,N,Kd", SHAPES)
def test_linear_many_tiles_bit_equal(M, N, Kd):
    torch.manual_seed(0)
    x = torch.randn(M, Kd, device="cuda").to(BF)
    w = (torch.randn(N, Kd, device="cuda") * 0.1).to(BF)
    assert torch.equal(T.linear(x, w), torch.mm(x, w.t()))


@pytest.mark.parametrize("M,N,Kd", SHAPES)
def test_linear_nn_many_tiles_bit_equal(M, N, Kd):
    torch.manual_seed(1)
    a = torch.randn(M, Kd, device="cuda").to(BF)
    b = (torch.randn(Kd, N, device="cuda") * 0.1).to(BF)
    assert T.nn_usable(a, b)
    assert torch.equal(T.linear_nn(a, b), torch.mm(a, b))


def test_edge_tiles_leave_neighbours_untouched():
    torch.manual_seed(2)
    M, N, Kd = 1000, 200, 256
    x = torch.randn(M, Kd, device="cuda").to(BF)
    w = (torch.randn(N, Kd, device="cuda") * 0.1).to(BF)
    buf = torch.full((M + 64, 512), 7.0, device="cuda", dtype=BF)
    T.linear(x, w, buf[:M, 64:64 + N])
    assert torch.equal(buf[:M, 64:64 + N], torch.mm(x, w.t()))
    keep = torch.ones_like(buf, dtype=torch.bool)
    keep[:M, 64:64 + N] = False
    assert bool((buf[keep] == 7.0).all())            # left, right and below the view: not written


def test_swiglu_bench_shape():
    torch.manual_seed(3)
    M, I, Kd = 32768, 2688, 1024
    x = torch.randn(M, Kd, device="cuda").to(BF)
    w = (torch.randn(2 * I, Kd, device="cuda") * 0.1).to(BF)
    gu, act = torch.empty(M, 2 * I, device="cuda", dtype=BF), torch.empty(M, I, device="cuda", dtype=BF)
    T.linear_swiglu(x, w, gu, act)
    gu_ref = torch.mm(x, w.t())
    assert torch.equal(gu, gu_ref)
    g, u = gu_ref[:, :I].float(), gu_ref[:, I:].float()
    assert rel(act, torch.nn.functional.silu(g) * u) < 4e-3


def test_qkv_rope_bench_shape():
    torch.manual_seed(4)
    B, S, H, Kd = 32, 1024, 16, 1024
    M, N = B * S, 3 * H * 64
    x = torch.randn(M, Kd, device="cuda").to(BF)
    w = (torch.randn(N, Kd, device="cuda") * 0.1).to(BF)
    cos, sin = K.rope_tables(S, 64, 10000.0, "cuda")
    ref = torch.mm(x, w.t())
    v_ref = ref[:, 2 * H * 64:].clone()
    K.rope_(ref, cos, sin, S, 2 * H, 64)
    out = torch.empty_like(ref)
    T.linear_qkv_rope(x, w, out, cos, sin, S, 2 * H * 64)
    assert rel(out, ref) < 1e-3
    assert torch.equal(out[:, 2 * H * 64:], v_ref)


@pytest.mark.parametrize("N,Kd", [(1024, 1024), (1000, 520)])
def test_wgrad_split_k_beyond_grid(N, Kd):
    torch.manual_seed(5)
    Tn = 32768
    dy = torch.randn(Tn, N, device="cuda").to(BF)
    x = torch.randn(Tn, Kd, device="cuda").to(BF)
    acc = torch.randn(N, Kd, device="cuda")
    step = dy.double().t() @ x.double()
    ref = acc.double() + step
    T.wgrad_acc(dy, x, acc)
    assert rel(acc, ref) < 2e-5
    T.wgrad_acc(dy, x, acc)
    assert rel(acc, ref + step) < 2e-5


def test_output_feeds_next_gemm():
    """The second GEMM reads the first one's TMA-stored output straight away on the same stream."""
    torch.manual_seed(6)
    M, Kd, N1, N2 = 32768, 1024, 1024, 3072
    x = torch.randn(M, Kd, device="cuda").to(BF)
    w1 = (torch.randn(N1, Kd, device="cuda") * 0.05).to(BF)
    w2 = (torch.randn(N2, N1, device="cuda") * 0.05).to(BF)
    h = torch.empty(M, N1, device="cuda", dtype=BF)
    for _ in range(3):
        h.fill_(0)
        T.linear(x, w1, h)
        y = T.linear(h, w2)
        assert torch.equal(y, torch.mm(torch.mm(x, w1.t()), w2.t()))


def test_misaligned_output_falls_back():
    torch.manual_seed(7)
    M, N, Kd = 512, 256, 128
    x = torch.randn(M, Kd, device="cuda").to(BF)
    w = (torch.randn(N, Kd, device="cuda") * 0.1).to(BF)
    flat = torch.zeros(M * N + 1, device="cuda", dtype=BF)
    out = flat[1:].view(M, N)                       # base 2 bytes past an aligned address
    assert out.data_ptr() % 16 != 0 and not T.usable(out) and not T.nn_usable(x, w.t().contiguous(), out)
    G.mm_nt(x, w, out)                              # the library GEMM (its kernel choice for a misaligned output may differ)
    assert rel(out, x.float() @ w.float().t()) < 4e-3
    out.zero_()
    G.mm_nn(x, w.t().contiguous(), out)
    assert rel(out, x.float() @ w.float().t()) < 4e-3
    acc = torch.zeros(N * 64 + 1, device="cuda")[1:].view(N, 64)     # fp32 dW 4 bytes past an aligned address
    G.mm_tn_acc(torch.randn(M, N, device="cuda").to(BF), torch.randn(M, 64, device="cuda").to(BF), acc)
    assert acc.abs().sum() > 0
