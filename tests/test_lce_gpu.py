"""Fused linear-cross-entropy (wgmma GEMM with the exponentials in the epilogue; csrc/gemm_sm90.cu kLCEFwd / kLCEdX,
csrc/lce.cu) against a plain fp32 PyTorch cross-entropy of the same op (reference call site train_diloco_torch.py:313-314)."""
import pytest
import torch

from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import gemm as G
from opendiloco_b200.ops import kernels as K
from opendiloco_b200.ops import tc_gemm as T

pytestmark = pytest.mark.gpu
BF = torch.bfloat16


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


def fused_lce(x, w, labels, loss_scale, train=True, want_norm=False):
    """Drive the kernels exactly as LlamaEngine._head_loss_fused does (labels already shifted)."""
    Tn, h = x.shape
    V = w.shape[0]
    dev = x.device
    planes = T.lce_planes(V)
    n_valid = (labels >= 0).sum().clamp(min=1).float().reshape(1)
    gscale = (loss_scale / n_valid).float()
    loss_sum = torch.zeros(1, device=dev)
    sumsq = torch.zeros(1, device=dev) if want_norm else None
    shift = torch.empty(Tn, device=dev)
    rowscale = torch.empty(Tn, device=dev)
    partials = torch.empty(2 * planes * Tn, device=dev)
    e = torch.empty(Tn, V, device=dev, dtype=BF) if train else None
    xs = torch.empty(Tn, h, device=dev, dtype=BF) if train else None
    dw = torch.zeros(V, h, device=dev) if train else None
    dx = torch.empty(Tn, h, device=dev, dtype=BF) if train else None
    K.lce_label_dot(x, w, labels, shift)
    T.lce_fwd(x, w, shift, partials, e, want_sumsq=want_norm)
    K.lce_finalize(partials, planes, labels, gscale, loss_sum, sumsq, rowscale if train else None, x, xs, dw)
    if train:
        T.lce_dx(e, w, rowscale, labels, gscale, dx)
        G.mm_tn_acc(e, xs, dw)
    return loss_sum / n_valid, dx, dw, sumsq


def reference_lce(x, w, labels, loss_scale):
    xf = x.float().requires_grad_(True)
    wf = w.float().requires_grad_(True)
    logits = xf @ wf.t()
    loss = torch.nn.functional.cross_entropy(logits, labels, ignore_index=-100, reduction="mean")
    (loss * loss_scale).backward()
    return loss.detach(), xf.grad, wf.grad, logits.detach().pow(2).sum()


@pytest.mark.parametrize("Tn,V,h,scale", [(256, 512, 64, 1.0), (300, 1000, 128, 0.25), (4096, 32000, 1024, 1.0)])
def test_fused_lce_matches_fp32(Tn, V, h, scale):
    torch.manual_seed(0)
    x = torch.randn(Tn, h, device="cuda").to(BF)
    w = (torch.randn(V, h, device="cuda") * (2.0 / h ** 0.5)).to(BF)        # logits of a few units: a peaked softmax
    labels = torch.randint(0, V, (Tn,), device="cuda")
    labels[::7] = -100
    loss, dx, dw, sumsq = fused_lce(x, w, labels, scale, want_norm=True)
    rloss, rdx, rdw, rsq = reference_lce(x, w, labels, scale)
    assert abs(loss.item() - rloss.item()) / rloss.item() < 1e-4
    assert rel(dx, rdx) < 5e-3
    assert rel(dw, rdw) < 5e-3
    assert abs(sumsq.item() - rsq.item()) / rsq.item() < 1e-3
    assert torch.count_nonzero(dx[::7]) == 0                                  # ignored rows: exactly zero gradient
    # evaluation mode: nothing of size [T, V] is written, same loss
    eloss, _, _, _ = fused_lce(x, w, labels, scale, train=False)
    assert abs(eloss.item() - rloss.item()) / rloss.item() < 1e-4


def test_fused_lce_flagship_shape():
    """T = 32768 tokens (32 x 1024), V = 32000, h = 1024: the Llama-150M micro-batch of the benchmark."""
    torch.manual_seed(1)
    Tn, V, h = 32768, 32000, 1024
    x = torch.randn(Tn, h, device="cuda").to(BF)
    w = (torch.randn(V, h, device="cuda") * 0.02).to(BF)
    labels = torch.randint(0, V, (Tn,), device="cuda")
    labels[1023::1024] = -100
    loss, dx, dw, _ = fused_lce(x, w, labels, 1.0 / 16)
    # fp32 reference in row chunks (the fp32 logits of the whole micro-batch would be 4.2 GB)
    n_valid = (labels >= 0).sum().item()
    rloss = 0.0
    rdx = torch.empty(Tn, h, device="cuda")
    rdw = torch.zeros(V, h, device="cuda")
    wf = w.float()
    for c0 in range(0, Tn, 4096):
        xf = x[c0:c0 + 4096].float()
        lab = labels[c0:c0 + 4096]
        lg = xf @ wf.t()
        lse = torch.logsumexp(lg, -1)
        valid = lab >= 0
        rloss += ((lse - lg.gather(1, lab.clamp(min=0)[:, None])[:, 0]) * valid).sum().item()
        p = torch.softmax(lg, -1)
        p.scatter_add_(1, lab.clamp(min=0)[:, None], -torch.ones_like(p[:, :1]))
        p *= (valid[:, None] / (16.0 * n_valid))
        rdx[c0:c0 + 4096] = p @ wf
        rdw += p.t() @ xf
    rloss /= n_valid
    assert abs(loss.item() - rloss) / rloss < 1e-4
    assert rel(dx, rdx) < 5e-3
    assert rel(dw, rdw) < 5e-3


def test_fused_lce_extreme_logits():
    """Label far below the best logit (loss of tens of nats) and large-magnitude logits: the shifted exponentials stay
    finite and the result still matches fp32."""
    torch.manual_seed(2)
    Tn, V, h = 512, 2048, 128
    x = (torch.randn(Tn, h, device="cuda") * 3).to(BF)
    w = (torch.randn(V, h, device="cuda") * 0.3).to(BF)                     # logits ~ N(0, 10^2): best - label up to ~80 nats
    labels = torch.randint(0, V, (Tn,), device="cuda")
    loss, dx, dw, _ = fused_lce(x, w, labels, 1.0)
    rloss, rdx, rdw, _ = reference_lce(x, w, labels, 1.0)
    assert torch.isfinite(dx.float()).all() and torch.isfinite(dw).all()
    assert rloss.item() > 25                                                  # the regime is extreme: mean loss of tens of nats
    assert abs(loss.item() - rloss.item()) / rloss.item() < 1e-4            # head-room: best logit up to 109 nats above the label
    assert rel(dx, rdx) < 5e-3 and rel(dw, rdw) < 5e-3


def test_engine_head_uses_fused_path_and_matches_reference(monkeypatch):
    """LlamaEngine.head_loss: fused path vs the materialising reference path on the same weights."""
    torch.manual_seed(3)
    cfg = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4, vocab_size=3000)
    ids = torch.randint(3, 3000, (4, 256), device="cuda")
    out = {}
    for mode in ("1", "0"):
        monkeypatch.setenv("ODB_LCE_FUSED", mode)
        m = LlamaForCausalLM(cfg, device="cuda", seed=5)
        loss = m.forward_backward(ids, ids, 0.5)
        out[mode] = (loss.item(), m.arena.grad.clone())
        ws = next(iter(m.engine._ws.values()))
        assert (ws._logits is None) == (mode == "1")                          # the fused path never allocates a logits tile
    assert abs(out["1"][0] - out["0"][0]) < 2e-3
    assert rel(out["1"][1], out["0"][1]) < 1e-2
