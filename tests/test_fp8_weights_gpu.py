"""FP8 weight-only generation on the sm_90a kernels: the per-row quantiser bit for bit against the reference, the skinny-M
e4m3 GEMM row by row against fp64, and ``generate(fp8_weights=True)`` end to end at the 150m and 1b shapes against the
bf16 program on the dequantised weights Ŵ."""
import json
import os
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from opendiloco_b200.models import fp8_weights as W8
from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.generation import decode_state
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import fp8w as FW
from opendiloco_b200.ops import tc_gemm as TC

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = Path(ROOT) / "opendiloco_b200" / "csrc"
DEV = "cuda"
FIRST = {"qkv": "self_attn.q_proj.weight", "o": "self_attn.o_proj.weight", "gu": "mlp.gate_proj.weight",
         "down": "mlp.down_proj.weight"}


def _shapes(name):
    c = LlamaConfig.from_pretrained(name)
    return {"qkv": (c.qkv_dim, c.hidden_size), "o": (c.hidden_size, c.q_dim), "gu": (2 * c.intermediate_size, c.hidden_size),
            "down": (c.hidden_size, c.intermediate_size)}


def _weights(N, K, seed, inject=True):
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = (torch.randn(N, K, generator=g, device=DEV) * 0.02).to(torch.bfloat16)
    if inject:
        w[3] = 0                                      # zero row
        w[5] *= 1e4                                   # huge row
        w[7] *= 1e-30                                 # tiny row
        w[11, 17] = float("nan")                      # NaN row
        w[13, 1] = 3.5                                # a row whose amax lands exactly on 448
    return w


def _nan_equal(a, b):
    return torch.equal(a.isnan(), b.isnan()) and torch.equal(a.nan_to_num(), b.nan_to_num())


# ------------------------------------------------------------------------------------------------ quantiser
@pytest.mark.parametrize("preset", ["150m", "1b"])
def test_quantizer_bit_identical(preset):
    shapes = _shapes(preset)
    ws = [_weights(N, K, i) for i, (N, K) in enumerate(shapes.values())]
    q = [torch.full(w.shape, 0x55, dtype=torch.uint8, device=DEV) for w in ws]
    inv = [torch.full((w.shape[0],), 7.0, device=DEV) for w in ws]
    deq = [torch.full_like(w, 7.0) for w in ws]
    segs = torch.tensor([[w.data_ptr(), a.data_ptr(), b.data_ptr(), c.data_ptr(), w.shape[0], w.shape[1]]
                         for w, a, b, c in zip(ws, q, inv, deq)], dtype=torch.int64, device=DEV)
    FW.quantize_rows(segs, len(ws), max(w.shape[0] for w in ws), ws[0])
    torch.cuda.synchronize()
    for w, qk, ik, dk in zip(ws, q, inv, deq):
        qr, ir = FW.quantize_rows_ref(w)
        assert torch.equal(qk, qr.view(torch.uint8))
        assert _nan_equal(ik, ir)
        assert _nan_equal(dk, FW.dequantize_rows(qr, ir))
        assert bool(torch.isnan(ik[11])) and float(ik[3]) == 1.0


# ------------------------------------------------------------------------------------------------ skinny GEMM
def _gemm_case(N, K, M, seed):
    w = _weights(N, K, seed, inject=False)
    q, inv = FW.quantize_rows_ref(w)
    x = (torch.randn(M, K, generator=torch.Generator(device=DEV).manual_seed(seed + 1), device=DEV)).to(torch.bfloat16)
    return x, q, inv, FW.dequantize_rows(q, inv)


def _check_rows(y, x, deq, K):
    """Row by row against fp64: |y - ref| <= 2^-8 |ref| (the bf16 output rounding) + K * 2^-24 * sum |x| |Ŵ| (fp32
    accumulation in any order)."""
    xd, wd = x.double(), deq.double()
    ref = xd @ wd.t()
    mag = xd.abs() @ wd.abs().t()
    err = (y.double() - ref).abs()
    tol = 2.0 ** -8 * ref.abs() + K * 2.0 ** -24 * mag
    bad = err > tol
    assert not bool(bad.any()), (int(bad.sum()), float((err - tol).max()))


def _run(x, q, inv, splits, act=None):
    N = q.shape[0]
    out = torch.full((x.shape[0], N), float("nan"), dtype=torch.bfloat16, device=DEV)
    ws = torch.zeros(max(FW.workspace_floats(N, splits), 1), device=DEV)
    cnt = torch.zeros(N // FW.TILE_N, dtype=torch.int32, device=DEV)
    FW.linear(x, q, inv, out, splits, ws, cnt, act=act)
    return out, cnt


@pytest.mark.parametrize("preset", ["60m", "150m", "1b"])
@pytest.mark.parametrize("kind", ["qkv", "o", "gu", "down"])
def test_skinny_gemm_against_fp64(preset, kind):
    N, K = _shapes(preset)[kind]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    default = FW.default_splits(N, K, sms)
    for M in range(1, 65):
        x, q, inv, deq = _gemm_case(N, K, M, M)
        for splits in ({1, default, K // FW.SPLIT_UNIT} if M in (1, 7, 8, 9, 33, 64) else {default}):
            y, cnt = _run(x, q, inv, splits)
            _check_rows(y, x, deq, K)
            assert not bool(cnt.any())                # the arrival counters are back at zero


@pytest.mark.parametrize("preset", ["150m", "1b"])
def test_skinny_swiglu_epilogue(preset):
    N, K = _shapes(preset)["gu"]
    I = N // 2
    for M in (1, 8, 13, 64):
        x, q, inv, deq = _gemm_case(N, K, M, 100 + M)
        act = torch.empty(M, I, dtype=torch.bfloat16, device=DEV)
        gu, _ = _run(x, q, inv, 3, act=act)
        _check_rows(gu, x, deq, K)
        g, u = gu[:, :I].float(), gu[:, I:].float()
        assert torch.allclose(act.float(), g * torch.sigmoid(g) * u, rtol=2.0 ** -6, atol=1e-6)
        # where the bf16 SwiGLU GEMM on Ŵ rounds gate and up identically, act is the same bits: the same formula
        gu_ref, act_ref = torch.empty_like(gu), torch.empty_like(act)
        TC.linear_swiglu(x, deq, gu_ref, act_ref)
        same = (gu_ref[:, :I] == gu[:, :I]) & (gu_ref[:, I:] == gu[:, I:])
        assert float(same.float().mean()) > 0.5
        assert torch.equal(act[same], act_ref[same])


def test_skinny_gemm_deterministic():
    N, K = _shapes("1b")["down"]
    x, q, inv, _ = _gemm_case(N, K, 24, 5)
    first, _ = _run(x, q, inv, 9)
    for _ in range(4):
        again, _ = _run(x, q, inv, 9)
        assert torch.equal(again, first)


# ------------------------------------------------------------------------------------------------ end to end
def master_view(ar, kind, l):
    N, K = W8.arena_weight(ar, kind, l).shape
    s = ar.slots[f"model.layers.{l}.{FIRST[kind]}"]
    return ar.master[s.offset:s.offset + N * K].view(N, K)


def what_copy(model):
    cp = LlamaForCausalLM(model.config, device=DEV, precision="bf16-mixed", init=False)
    cp.arena.master.copy_(model.arena.master)
    cp.arena.sync_shadow()
    for kind in W8.KINDS:
        for l in range(model.config.num_hidden_layers):
            q, inv = FW.quantize_rows_ref(W8.arena_weight(model.arena, kind, l))
            master_view(cp.arena, kind, l).copy_(FW.dequantize_rows(q, inv, torch.float32))
    cp.arena.sync_shadow()
    return cp


_MODELS = {}


def _model(preset):
    if preset not in _MODELS:
        _MODELS.clear()
        cfg = LlamaConfig.from_pretrained(preset)
        if preset == "1b":
            cfg.num_hidden_layers = 6                 # the 1b shapes; fewer layers keep the test short
        m = LlamaForCausalLM(cfg, device=DEV, precision="bf16-mixed", seed=3)
        _MODELS[preset] = (m, what_copy(m))
    return _MODELS[preset]


def _agree_until_near_tie(judge, got, ref, P, gap=0.05):
    """Rows agree token for token up to the first step where the judge's top-2 logits are within ``gap``."""
    with torch.no_grad():
        logits = judge(ref).logits.float()
    top2 = logits[:, P - 1:-1].topk(2, dim=-1).values
    close = (top2[..., 0] - top2[..., 1]) < gap
    n = ref.shape[1] - P
    for b in range(ref.shape[0]):
        stop = int(torch.nonzero(close[b])[0]) if bool(close[b].any()) else n
        assert torch.equal(got[b, :P + stop], ref[b, :P + stop]), b


def _ids(V, B, P, seed=0):
    return torch.randint(3, V, (B, P), generator=torch.Generator().manual_seed(seed)).to(DEV)


@pytest.mark.parametrize("preset", ["150m", "1b"])
@pytest.mark.parametrize("B", [1, 8])
def test_greedy_matches_what_program(preset, B, monkeypatch):
    m, cp = _model(preset)
    ids = _ids(m.config.vocab_size, B, 40, B)
    got = m.generate(ids, max_new_tokens=24, eos_token_id=[], fp8_weights=True)
    ref = cp.generate(ids, max_new_tokens=24, eos_token_id=[])
    _agree_until_near_tie(cp, got, ref, 40)
    monkeypatch.setenv("ODB_CUDA_GRAPH", "0")
    eager = m.generate(ids, max_new_tokens=24, eos_token_id=[], fp8_weights=True)
    assert torch.equal(eager, got)                    # graph and eager: the same kernels, bit for bit


def test_toggle_recaptures_and_requantises():
    m, cp = _model("150m")
    ids = _ids(m.config.vocab_size, 4, 32, 7)
    plain = m.generate(ids, max_new_tokens=20, eos_token_id=[])
    fp8 = m.generate(ids, max_new_tokens=20, eos_token_id=[], fp8_weights=True)
    key8 = m.engine.decode_state.graph_key
    assert key8[-1] == m.engine.fp8_weights.token and m.engine.decode_state.graph is not None
    assert torch.equal(m.generate(ids, max_new_tokens=20, eos_token_id=[]), plain)
    assert m.engine.decode_state.graph_key[-1] is None
    assert torch.equal(m.generate(ids, max_new_tokens=20, eos_token_id=[], fp8_weights=True), fp8)
    # an optimizer-like in-place update: the next call quantises the new weights into the same buffers
    fw = m.engine.fp8_weights
    ptrs = {k: fw.q[k].data_ptr() for k in W8.KINDS}
    saved = m.arena.master.clone()
    try:
        with torch.no_grad():
            m.arena.master.mul_(1.5)
            m.arena.sync_shadow()
        changed = m.generate(ids, max_new_tokens=20, eos_token_id=[], fp8_weights=True)
        assert m.engine.fp8_weights is fw and {k: fw.q[k].data_ptr() for k in W8.KINDS} == ptrs
        q, inv = FW.quantize_rows_ref(W8.arena_weight(m.arena, "down", 1))
        assert torch.equal(fw.q["down"][1].view(torch.uint8), q.view(torch.uint8)) and _nan_equal(fw.inv["down"][1], inv)
        assert not torch.equal(changed, fp8)
    finally:
        with torch.no_grad():
            m.arena.master.copy_(saved)
            m.arena.sync_shadow()


def test_modes_run_with_fp8_weights():
    m, cp = _model("150m")
    V = m.config.vocab_size
    ids = _ids(V, 4, 48, 9)
    ids[:, 24:40] = ids[:, 0:16]                      # something for prompt lookup to find
    # prompt lookup at B 16, K 7: a 128-row verify pass takes the Ŵ GEMM, and prefill does too: the same bits as Ŵ
    wide = ids.repeat(4, 1)
    got = m.generate(wide, max_new_tokens=16, eos_token_id=[], prompt_lookup_num_tokens=7, fp8_weights=True)
    ref = cp.generate(wide, max_new_tokens=16, eos_token_id=[], prompt_lookup_num_tokens=7)
    assert torch.equal(got, ref)
    # narrow lookup (40-row verify: the skinny GEMM), assisted with the bf16 model as its own draft, and beam search
    plain = m.generate(ids, max_new_tokens=16, eos_token_id=[], fp8_weights=True)
    for kw in ({"prompt_lookup_num_tokens": 4}, {"assistant_model": m, "num_assistant_tokens": 3}):
        out = m.generate(ids, max_new_tokens=16, eos_token_id=[], fp8_weights=True, **kw)
        _agree_until_near_tie(cp, out, plain, 48)
    got = m.generate(ids, max_new_tokens=12, eos_token_id=[], num_beams=4, return_dict_in_generate=True, fp8_weights=True)
    ref = cp.generate(ids, max_new_tokens=12, eos_token_id=[], num_beams=4, return_dict_in_generate=True)
    assert got.sequences.shape == ref.sequences.shape
    assert torch.allclose(got.sequences_scores, ref.sequences_scores, atol=0.05, rtol=0)
    assert m.engine.beam_state.graph is not None and m.engine.beam_state.graph_key[-1] == m.engine.fp8_weights.token


def test_score_matches_what_model():
    m, cp = _model("150m")
    ids = _ids(m.config.vocab_size, 2, 200, 4)
    got, ref = m.score(ids, fp8_weights=True), cp.score(ids)
    assert torch.equal(got.logprobs, ref.logprobs)     # M > 64 everywhere: the bf16 GEMMs on Ŵ


def test_training_state_untouched():
    m, _ = _model("150m")
    ids = _ids(m.config.vocab_size, 2, 256, 1)
    m.forward_backward(ids, ids)
    graphs, wss = dict(m.engine._graphs), dict(m.engine._ws)
    before = {n: getattr(m.arena, n).clone() for n in ("master", "shadow", "grad")}
    m.generate(ids[:, :64], max_new_tokens=8, fp8_weights=True)
    m.score(ids, fp8_weights=True)
    for n, t in before.items():
        assert torch.equal(getattr(m.arena, n).view(torch.uint8), t.view(torch.uint8)), n
    assert m.engine._graphs == graphs and m.engine._ws == wss
    m.arena.grad.zero_()


_PROFILE_STEP = r"""
import json, os, sys
import torch
sys.path.insert(0, os.getcwd())
from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.generation import step
from opendiloco_b200.models.llama import LlamaForCausalLM
cfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=2, num_attention_heads=16, vocab_size=32000)
m = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=1)
ids = torch.randint(3, 32000, (8, 64), device="cuda")
m.generate(ids, max_new_tokens=4, eos_token_id=[], fp8_weights=True)
st, fw = m.engine.decode_state, m.engine.fp8_weights
from torch.profiler import ProfilerActivity, profile
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    step(m, st, graph=False, fp8=fw)
    torch.cuda.synchronize()
print(json.dumps({"gpu": [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]}))
"""


def test_decode_step_runs_only_our_kernels():
    ours = set()
    for src in CSRC.glob("*.cu"):
        ours |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(", src.read_text()))
    assert "fp8w_gemm_kernel" in ours
    res = subprocess.run([sys.executable, "-c", _PROFILE_STEP], capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    gpu = json.loads(res.stdout.strip().splitlines()[-1])["gpu"]
    assert gpu
    foreign = [n for n in gpu if not any(re.search(rf"\b{k}\b", n) for k in ours)]
    assert not foreign, foreign
    assert sum("fp8w_gemm_kernel" in n for n in gpu) == 2 * 4      # every projection of both layers
