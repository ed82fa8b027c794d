"""Numerics of every sm_90a kernel against a plain PyTorch fp32 reference of the same op (run on an H100)."""
import math

import pytest
import torch

from opendiloco_b200.ops import attention as A
from opendiloco_b200.ops import gemm as G
from opendiloco_b200.ops import kernels as K

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


@pytest.fixture(autouse=True)
def _seed():
    torch.manual_seed(0)


def test_native_library_loaded():
    from opendiloco_b200 import _lib

    lib = _lib.cuda_lib()
    assert hasattr(lib, "odb_adamw_step")


@pytest.mark.parametrize("h", [64, 1024, 2048, 4096])
def test_embedding(h):
    V, T = 1000, 777
    W = torch.randn(V, h, device=DEV).to(BF)
    ids = torch.randint(0, V, (T,), device=DEV)
    out = K.embedding_fwd(ids, W)
    assert torch.equal(out, W[ids])
    dW = torch.zeros(V, h, device=DEV)
    dout = torch.randn(T, h, device=DEV).to(BF)
    K.embedding_bwd(ids, dout, dW)
    ref = torch.zeros(V, h, device=DEV).index_add_(0, ids, dout.float())
    assert rel(dW, ref) < 1e-5


@pytest.mark.parametrize("h", [64, 128, 1024, 2048, 4096])
@pytest.mark.parametrize("with_delta", [False, True])
def test_rmsnorm_fwd_bwd(h, with_delta):
    T = 515
    x = torch.randn(T, h, device=DEV).to(BF)
    d = torch.randn(T, h, device=DEV).to(BF) if with_delta else None
    w = (1 + 0.1 * torch.randn(h, device=DEV)).to(BF)
    xo = torch.empty_like(x)
    y, rstd = K.rmsnorm_fwd(x, w, 1e-5, delta=d, x_out=xo)
    xr = (x.float() + d.float()).to(BF).float() if with_delta else x.float()
    r = torch.rsqrt(xr.pow(2).mean(-1) + 1e-5)
    yref = w.float() * (xr * r[:, None]).to(BF).float()
    if with_delta:
        assert torch.equal(xo, xr.to(BF))
    assert rel(rstd, r) < 1e-5
    assert rel(y, yref) < 5e-3
    # backward against autograd in fp32
    xin = xr.clone().requires_grad_(True)
    wf = w.float().clone().requires_grad_(True)
    yy = wf * (xin * torch.rsqrt(xin.pow(2).mean(-1, keepdim=True) + 1e-5))
    dy = torch.randn(T, h, device=DEV).to(BF)
    yy.backward(dy.float())
    dres = torch.randn(T, h, device=DEV).to(BF)
    dres_out = torch.empty_like(dres)
    dw = torch.zeros(h, device=DEV)
    K.rmsnorm_bwd(dy, xr.to(BF), w, rstd, dres, dres_out, dw)
    assert rel(dres_out, dres.float() + xin.grad) < 6e-3
    assert rel(dw, wf.grad) < 6e-3


@pytest.mark.parametrize("D,Hq,Hkv", [(64, 16, 16), (64, 32, 4), (32, 2, 2)])
def test_rope(D, Hq, Hkv):
    B, S = 3, 128
    row = (Hq + 2 * Hkv) * D
    qkv = torch.randn(B * S, row, device=DEV).to(BF)
    cos, sin = K.rope_tables(S, D, 10000.0, DEV)
    ref = K.rope_(qkv.cpu().clone(), cos.cpu(), sin.cpu(), S, Hq + Hkv, D)
    out = K.rope_(qkv.clone(), cos, sin, S, Hq + Hkv, D)
    assert rel(out, ref.to(DEV)) < 4e-3
    assert torch.equal(out[:, (Hq + Hkv) * D:], qkv[:, (Hq + Hkv) * D:])          # v untouched
    back = K.rope_(out.clone(), cos, sin, S, Hq + Hkv, D, backward=True)          # rotation is orthogonal
    assert rel(back, qkv) < 1e-2


@pytest.mark.parametrize("I", [256, 2688, 5632])
def test_swiglu(I):
    T = 300
    gu = torch.randn(T, 2 * I, device=DEV).to(BF)
    a = K.swiglu_fwd(gu)
    g, u = gu[:, :I].float(), gu[:, I:].float()
    assert rel(a, torch.nn.functional.silu(g) * u) < 4e-3
    da = torch.randn(T, I, device=DEV).to(BF)
    gg, uu = g.clone().requires_grad_(True), u.clone().requires_grad_(True)
    (torch.nn.functional.silu(gg) * uu).backward(da.float())
    dgu = K.swiglu_bwd(da, gu)
    assert rel(dgu[:, :I], gg.grad) < 5e-3 and rel(dgu[:, I:], uu.grad) < 5e-3


@pytest.mark.parametrize("V", [1024, 32000, 50264])
def test_cross_entropy(V):
    R = 257
    logits = (3 * torch.randn(R, V, device=DEV)).to(BF)
    labels = torch.randint(0, V, (R,), device=DEV)
    labels[::7] = -100
    x = logits.float().clone().requires_grad_(True)
    loss_ref = torch.nn.functional.cross_entropy(x, labels, ignore_index=-100, reduction="sum")
    loss_ref.backward()
    gscale = torch.tensor([0.37], device=DEV)
    loss_sum = torch.zeros(1, device=DEV)
    sumsq = torch.zeros(1, device=DEV)
    work = logits.clone()
    K.ce_fwd_bwd_(work, labels, gscale, loss_sum, sumsq)
    assert abs(loss_sum.item() - loss_ref.item()) / abs(loss_ref.item()) < 2e-3
    assert rel(work, x.grad * 0.37) < 1e-2
    assert abs(sumsq.item() - logits.float().pow(2).sum().item()) / sumsq.item() < 1e-3
    l2 = torch.zeros(1, device=DEV)
    K.ce_fwd(logits, labels, l2)
    assert abs(l2.item() - loss_ref.item()) / abs(loss_ref.item()) < 2e-3


def test_adamw_matches_torch():
    n = 1 << 20
    p0 = torch.randn(n, device=DEV)
    g0 = torch.randn(n, device=DEV) * 0.01
    ref_p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.AdamW([ref_p], lr=4e-4, weight_decay=0.1, betas=(0.9, 0.95))
    p, m, v = p0.clone(), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    shadow = torch.zeros(n, device=DEV, dtype=BF)
    hp = torch.zeros(K.HP_SIZE, device=DEV)
    partials = torch.zeros(K.MAX_PARTIALS, device=DEV)
    flag = torch.zeros(1, device=DEV, dtype=torch.int32)
    stats = torch.zeros(2, device=DEV)
    for step in range(1, 4):
        g = g0 * step
        ref_p.grad = g.clone()
        tot = torch.nn.utils.clip_grad_norm_([ref_p], 1.0)
        opt.step()
        gg = g.clone()
        npart = K.grad_sqnorm(gg, partials, flag)
        hp[:9] = torch.tensor([4e-4, 0.9, 0.95, 1e-8, 0.1, 1 - 0.9 ** step, 1 - 0.95 ** step, 1.0, 1.0], device=DEV)
        K.adamw_step(p, gg, m, v, shadow, hp, partials, npart, None, stats, zero_grad=True)
        assert abs(stats[0].item() - tot.item()) / tot.item() < 1e-4
        assert torch.count_nonzero(gg) == 0
        assert (p - ref_p.data).abs().max().item() < 2e-6
        assert torch.equal(shadow, p.to(BF))
    assert flag.item() == 0


@pytest.mark.parametrize("delta_dtype", [None, torch.float32, BF])
def test_nesterov_outer_matches_torch_sgd(delta_dtype):
    n = 1 << 18
    theta_outer = torch.randn(n, device=DEV)
    theta_local = theta_outer + 0.01 * torch.randn(n, device=DEV)
    ref = torch.nn.Parameter(theta_outer.clone())
    sgd = torch.optim.SGD([ref], lr=0.7, momentum=0.9, nesterov=True)
    buf = torch.zeros(n, device=DEV)
    shadow = torch.zeros(n, device=DEV, dtype=BF)
    to, tl = theta_outer.clone(), theta_local.clone()
    for _ in range(3):
        d = to - tl
        if delta_dtype is None:
            delta = None
        else:
            delta = torch.empty(n, device=DEV, dtype=delta_dtype)
            K.pseudo_grad(to, tl, delta)
            d = delta.float()
        ref.grad = d.clone()
        sgd.step()
        K.nesterov_outer(to, buf, delta, tl, shadow, 0.7, 0.9, True)
        tol = 1e-6 if delta_dtype != BF else 1e-6
        assert (to - ref.data).abs().max().item() < tol
        assert torch.equal(tl, to) and torch.equal(shadow, to.to(BF))
        tl = to + 0.01 * torch.randn(n, device=DEV)


@pytest.mark.parametrize("Hq,Hkv", [(16, 16), (32, 4)])
def test_attention_library_path(Hq, Hkv):
    B, S, D = 2, 256, 64
    qkv = torch.randn(B * S, (Hq + 2 * Hkv) * D, device=DEV).to(BF)
    out, aux = A.attention_fwd(qkv, B, S, Hq, Hkv, D)
    ref, _ = A.attention_fwd(qkv.cpu().float(), B, S, Hq, Hkv, D)
    assert rel(out, ref.to(DEV)) < 1e-2
    dout = torch.randn_like(out)
    dqkv = torch.empty_like(qkv)
    A.attention_bwd(dout, qkv, out, aux, dqkv, B, S, Hq, Hkv, D)
    qc = qkv.cpu().float()
    oc, auxc = A.attention_fwd(qc, B, S, Hq, Hkv, D)
    dref = torch.empty_like(qc)
    A.attention_bwd(dout.cpu().float(), qc, oc, auxc, dref, B, S, Hq, Hkv, D)
    assert rel(dqkv, dref.to(DEV)) < 2e-2


def test_wgrad_fp32_accumulate():
    T, N, Kd = 512, 256, 384
    a = torch.randn(T, N, device=DEV).to(BF)
    b = torch.randn(T, Kd, device=DEV).to(BF)
    acc = torch.randn(N, Kd, device=DEV)
    ref = acc + a.float().t() @ b.float()
    G.mm_tn_acc(a, b, acc)
    assert rel(acc, ref) < 1e-3


@pytest.mark.parametrize("B,S,Hq,Hkv", [(1, 128, 1, 1), (2, 256, 4, 2), (2, 1024, 4, 4), (3, 512, 8, 1)])
def test_tcgen05_attention_forward(B, S, Hq, Hkv):
    """Our causal attention forward (csrc/attn_sm90.cu) against the fp32 math reference."""
    qkv = torch.randn(B * S, (Hq + 2 * Hkv) * 64, device=DEV).to(BF)
    out, lse = A.tc_attention_fwd(qkv, B, S, Hq, Hkv)
    ref, (lse_ref, _) = A.attention_fwd(qkv.float(), B, S, Hq, Hkv, 64)
    assert rel(out, ref) < 5e-3
    assert (lse - lse_ref).abs().max().item() < 1e-3


@pytest.mark.parametrize("B,S,Hq,Hkv", [(1, 128, 1, 1), (2, 256, 4, 2), (1, 384, 2, 1), (2, 1024, 4, 4), (2, 512, 8, 1)])
def test_tcgen05_attention_backward(B, S, Hq, Hkv):
    """Our attention backward (csrc/attn_bwd_sm90.cu: pre-pass, main kernel, post-pass) against the fp32 math
    reference; S = 384 is not a multiple of 256."""
    qkv = torch.randn(B * S, (Hq + 2 * Hkv) * 64, device=DEV).to(BF)
    out, lse = A.tc_attention_fwd(qkv, B, S, Hq, Hkv)
    dout = torch.randn_like(out)
    dq, dk, dv = A.tc_attention_bwd(dout, qkv, out, lse, B, S, Hq, Hkv)
    qf = qkv.float()
    of, aux = A.attention_fwd(qf, B, S, Hq, Hkv, 64)
    dref = torch.empty_like(qf)
    A.attention_bwd(dout.float(), qf, of, aux, dref, B, S, Hq, Hkv, 64)
    q_dim, kv_dim = Hq * 64, Hkv * 64
    assert rel(dq, dref[:, :q_dim]) < 1e-2
    assert rel(dk, dref[:, q_dim:q_dim + kv_dim]) < 1e-2
    assert rel(dv, dref[:, q_dim + kv_dim:]) < 1e-2


def test_tcgen05_attention_backward_packed_rope():
    """Packed output + fused RoPE-transpose post-pass == dense output followed by the stand-alone rope kernel."""
    B, S, Hq, Hkv = 2, 256, 4, 2
    qkv = torch.randn(B * S, (Hq + 2 * Hkv) * 64, device=DEV).to(BF)
    cos, sin = K.rope_tables(S, 64, 10000.0, torch.device(DEV))
    out, lse = A.tc_attention_fwd(qkv, B, S, Hq, Hkv)
    dout = torch.randn_like(out)
    dq, dk, dv = A.tc_attention_bwd(dout, qkv, out, lse, B, S, Hq, Hkv)
    ref = torch.cat([dq, dk, dv], dim=1).contiguous()
    K.rope_(ref, cos, sin, S, Hq + Hkv, 64, backward=True)
    packed = torch.zeros_like(ref)
    res = A.tc_attention_bwd(dout, qkv, out, lse, B, S, Hq, Hkv, dqkv=packed, cos=cos, sin=sin)
    assert res is packed
    assert rel(packed, ref) < 6e-3       # dq is rotated in fp32 before its single bf16 rounding; the reference rounds twice
    assert torch.equal(packed[:, (Hq + Hkv) * 64:], dv)


def test_grad_scaler_on_the_fused_kernel_path():
    """fp16-mixed bookkeeping on the kernels (K11): 1/scale as device-side hyper-parameter, non-finite flag from the norm
    pass, skipped update + halved scale on overflow (reference flow train_fsdp.py:390-405, utils.py:124-135)."""
    import copy

    from opendiloco_b200.optim.fused import FusedAdamW
    from opendiloco_b200.utils.training import found_inf_grad

    torch.manual_seed(0)
    ours = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.Linear(128, 32)).to(DEV)
    ref = copy.deepcopy(ours)
    opt = FusedAdamW(ours.parameters(), lr=1e-2, betas=(0.9, 0.95), weight_decay=0.1, max_grad_norm=1.0)
    ropt = torch.optim.AdamW(ref.parameters(), lr=1e-2, betas=(0.9, 0.95), weight_decay=0.1)
    scaler = torch.amp.GradScaler("cuda", init_scale=2048.0, growth_interval=1000)
    x = torch.randn(8, 64, device=DEV)
    for _ in range(3):
        scaler.scale(ours(x).pow(2).mean()).backward()
        ref(x).pow(2).mean().backward()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), 1.0)
        ropt.step()
        ropt.zero_grad()
        opt.unscale_(scaler)
        opt.step_scaled(scaler)
        assert not found_inf_grad(opt, scaler)
        scaler.update()
        opt.zero_grad()
        for p, q in zip(ours.parameters(), ref.parameters()):
            assert torch.allclose(p, q, atol=5e-6)
    before = [p.detach().clone() for p in ours.parameters()]
    scaler.scale(ours(x).pow(2).mean()).backward()
    next(ours.parameters()).grad[0, 0] = float("inf")
    opt.unscale_(scaler)
    opt.step_scaled(scaler)
    assert found_inf_grad(opt, scaler)
    s0 = scaler.get_scale()
    scaler.update()
    assert scaler.get_scale() == s0 * 0.5
    for p, q in zip(ours.parameters(), before):
        assert torch.equal(p, q)
