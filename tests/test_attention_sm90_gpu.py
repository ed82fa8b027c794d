"""Our sm_90a causal attention (csrc/attn_sm90.cu, csrc/attn_bwd_sm90.cu) at the shapes training runs: Llama-150M
(B32 S1024, 16 heads) and Llama-1B (B16 S1024, 32 query heads on 4 kv heads), against the fp32 math reference."""
import pytest
import torch

from opendiloco_b200.ops import attention as A
from opendiloco_b200.ops import kernels as K

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
SHAPES = [(32, 1024, 16, 16), (16, 1024, 32, 4)]


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _inputs(B, S, Hq, Hkv):
    torch.manual_seed(0)
    qkv = torch.randn(B * S, (Hq + 2 * Hkv) * 64, device=DEV).to(BF)
    out, lse = A.tc_attention_fwd(qkv, B, S, Hq, Hkv)
    dout = torch.randn_like(out)
    return qkv, out, lse, dout


@pytest.mark.parametrize("B,S,Hq,Hkv", SHAPES)
def test_forward_and_backward_at_training_shapes(B, S, Hq, Hkv):
    qkv, out, lse, dout = _inputs(B, S, Hq, Hkv)
    qf = qkv.float()
    ref, (lse_ref, _) = A.attention_fwd(qf, B, S, Hq, Hkv, 64)
    assert rel(out, ref) < 5e-3
    assert (lse - lse_ref).abs().max().item() < 1e-3
    del ref, lse_ref
    dq, dk, dv = A.tc_attention_bwd(dout, qkv, out, lse, B, S, Hq, Hkv)
    of, aux = A.attention_fwd(qf, B, S, Hq, Hkv, 64)
    dref = torch.empty_like(qf)
    A.attention_bwd(dout.float(), qf, of, aux, dref, B, S, Hq, Hkv, 64)
    q_dim, kv_dim = Hq * 64, Hkv * 64
    assert rel(dq, dref[:, :q_dim]) < 1e-2
    assert rel(dk, dref[:, q_dim:q_dim + kv_dim]) < 1e-2
    assert rel(dv, dref[:, q_dim + kv_dim:]) < 1e-2


def test_backward_packed_rope_at_flagship_shape():
    """The main kernel undoes RoPE on dK in its store and the post-pass on dQ: same as the dense output followed by
    the stand-alone inverse rotation."""
    B, S, Hq, Hkv = SHAPES[0]
    qkv, out, lse, dout = _inputs(B, S, Hq, Hkv)
    cos, sin = K.rope_tables(S, 64, 10000.0, torch.device(DEV))
    dq, dk, dv = A.tc_attention_bwd(dout, qkv, out, lse, B, S, Hq, Hkv)
    ref = torch.cat([dq, dk, dv], dim=1).contiguous()
    K.rope_(ref, cos, sin, S, Hq + Hkv, 64, backward=True)
    packed = torch.zeros_like(ref)
    res = A.tc_attention_bwd(dout, qkv, out, lse, B, S, Hq, Hkv, dqkv=packed, cos=cos, sin=sin)
    assert res is packed
    # dq and dk are rotated in fp32 before their single bf16 rounding; the reference rounds twice
    assert rel(packed, ref) < 6e-3
    assert torch.equal(packed[:, (Hq + Hkv) * 64:], dv)


@pytest.mark.parametrize("B,S,Hq,Hkv", SHAPES)
def test_backward_calls_reusing_scratch_agree(B, S, Hq, Hkv):
    """The dQ accumulator and statistics scratch is shared by every call: a second call must start from zero."""
    qkv, out, lse, dout = _inputs(B, S, Hq, Hkv)
    first = [t.clone() for t in A.tc_attention_bwd(dout, qkv, out, lse, B, S, Hq, Hkv)]
    second = A.tc_attention_bwd(dout, qkv, out, lse, B, S, Hq, Hkv)
    for a, b in zip(first, second):
        assert rel(b, a) < 1e-3           # only the order of the fp32 dQ reduce-adds varies between calls
    assert torch.equal(first[1], second[1]) and torch.equal(first[2], second[2])
