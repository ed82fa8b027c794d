"""FP8 KV cache on the sm_90a decode kernels (H100).

- Writers: the three FP8 cache writers store bytes and inv bit-identical to ``quantize_rows_ref`` of what the bf16
  writers store (and rotate q the same way), at the 150m and 1b head counts, with injected zero / huge / NaN heads.
- Readers: decode attention (G 1, 2, 4, 8; B up to 64; edge and ragged positions; with and without a chunk table) and
  verify attention (n = 1..8) on the FP8 cache equal the bf16 kernels on the dequantised cache Ĉ bit for bit.  The
  data stay above amax 448 * 2^-125, where Ĉ is a bf16 number.
- Beam reorder: bytes and inv, read through the chunk table, equal the physical reference reorder.
- End to end (60m, bf16-mixed): every generation mode, alone and with ``fp8_weights=True``, in eager and graph mode, gives
  exactly the tokens (and beam scores) of the eager oracle program of ``test_fp8_kv_cache_cpu``.  Toggling, cache
  memory and the kernels one FP8 decode step launches."""
import json
import os
import re
import subprocess
import sys
from pathlib import Path

import pytest
import torch

from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import decode as DK
from opendiloco_b200.ops import fp8w as FW
from opendiloco_b200.ops import kernels as K
from opendiloco_b200.ops.fp8 import E4M3
from test_fp8_kv_cache_cpu import oracle_generate

pytestmark = pytest.mark.gpu
DEV = "cuda"
D = 64
ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "opendiloco_b200" / "csrc"


def _nan_equal(a, b):
    return torch.equal(torch.nan_to_num(a, nan=-7.0), torch.nan_to_num(b, nan=-7.0)) and torch.equal(a.isnan(), b.isnan())


def _assert_rows(kq, ki, kb, written):
    """FP8 cache (kq, ki) == quantize_rows_ref of the bf16 cache kb in the written rows ([B, Hkv, Smax] bool)."""
    q, inv = FW.quantize_rows_ref(kb[written])
    assert torch.equal(kq.view(torch.uint8)[written], q.view(torch.uint8))
    assert _nan_equal(ki[written], inv)


def _caches(B, Hkv, Smax):
    z = lambda dt: torch.zeros(B, Hkv, Smax, D, dtype=dt, device=DEV)  # noqa: E731
    return z(torch.bfloat16), z(torch.bfloat16), z(E4M3), z(E4M3), torch.zeros(B, Hkv, Smax, device=DEV), \
        torch.zeros(B, Hkv, Smax, device=DEV)


def _qkv(rows, Hq, Hkv, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(rows, Hq + 2 * Hkv, D, device=DEV, generator=g) * torch.exp(torch.randn(rows, Hq + 2 * Hkv, 1, device=DEV, generator=g))
    x[0, Hq] = 0.0                                     # a zero k head
    x[min(1, rows - 1), Hq + Hkv] = 0.0                # a zero v head
    x[min(2, rows - 1), Hq + Hkv - 1, 5] = 1.0e30      # huge values
    x[min(3, rows - 1), -1, 7] = -3.0e38
    x[min(4, rows - 1), Hq, 3] = float("nan")          # NaN heads
    x[min(5, rows - 1), Hq + Hkv, 9] = float("nan")
    return x.reshape(rows, -1).bfloat16()


@pytest.mark.parametrize("preset", ["150m", "1b"])
def test_writers_bit_identical(preset):
    cfg = LlamaConfig.from_pretrained(preset)
    Hq, Hkv, B, Smax, n = cfg.num_attention_heads, cfg.num_key_value_heads, 8, 256, 5
    cos, sin = K.rope_tables(Smax + 128, D, cfg.rope_theta, DEV)
    pos = torch.tensor([0, 1, 127, 128, 129, 200, 31, Smax - n], dtype=torch.int32, device=DEV)
    for multi in (False, True):
        x = _qkv(n * B if multi else B, Hq, Hkv, 1 + multi)
        kb, vb, kq, vq, ki, vi = _caches(B, Hkv, Smax)
        a, b = x.clone(), x.clone()
        if multi:
            DK.rope_append_multi(a, cos, sin, pos, kb, vb, Hq, Hkv, D, n)
            DK.rope_append_multi(b, cos, sin, pos, kq, vq, Hq, Hkv, D, n, kinv=ki, vinv=vi)
        else:
            DK.rope_append(a, cos, sin, pos, kb, vb, Hq, Hkv, D)
            DK.rope_append(b, cos, sin, pos, kq, vq, Hq, Hkv, D, kinv=ki, vinv=vi)
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))               # the same rotated q
        w = torch.zeros(B, Hkv, Smax, dtype=torch.bool, device=DEV)
        for j in range(n if multi else 1):
            w[torch.arange(B, device=DEV), :, pos.long() + j] = True
        _assert_rows(kq, ki, kb, w)
        _assert_rows(vq, vi, vb, w)
        assert (ki[~w] == 0).all() and (kq.view(torch.uint8)[~w] == 0).all()
        assert bool(torch.isnan(ki).any()) and bool(torch.isnan(vi).any()) and bool((ki[w] == 1.0).any())
    # prefill, ragged lens, beam row stride 2
    Sp, Bp = 192, 4
    x = _qkv(Bp * Sp, Hq, Hkv, 7)
    lens = torch.tensor([192, 1, 130, 64], dtype=torch.int32, device=DEV)
    kb, vb, kq, vq, ki, vi = _caches(2 * Bp, Hkv, Smax)
    DK.kv_fill(x, lens, kb, vb, Bp, Sp, Hq, Hkv, D, row_stride=2)
    DK.kv_fill(x, lens, kq, vq, Bp, Sp, Hq, Hkv, D, row_stride=2, kinv=ki, vinv=vi)
    w = torch.zeros(2 * Bp, Hkv, Smax, dtype=torch.bool, device=DEV)
    for b in range(Bp):
        w[2 * b, :, :int(lens[b])] = True
    _assert_rows(kq, ki, kb, w)
    _assert_rows(vq, vi, vb, w)
    assert (ki[~w] == 0).all() and (vq.view(torch.uint8)[~w] == 0).all()


def _fp8_cache(B, Hkv, Smax, seed):
    """A random FP8 cache (bytes, inv) with row scales over many octaves, and its Ĉ."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    out = []
    for _ in range(2):
        x = (torch.randn(B, Hkv, Smax, D, device=DEV, generator=g)
             * torch.exp2(torch.randint(-20, 12, (B, Hkv, Smax, 1), device=DEV, generator=g).float())).bfloat16()
        q, inv = FW.quantize_rows_ref(x.view(-1, D))
        q, inv = q.view(x.shape), inv.view(x.shape[:-1])
        out.append((q, inv, FW.dequantize_rows(q.view(-1, D), inv.view(-1)).view(x.shape)))
    return out


def _positions(B, Smax, n, seed):
    edge = [0, 1, 127, 128, 129, Smax - n]
    g = torch.Generator().manual_seed(seed)
    rest = torch.randint(0, Smax - n + 1, (max(0, B - len(edge)),), generator=g).tolist()
    return torch.tensor((edge + rest)[:B], dtype=torch.int32, device=DEV)


@pytest.mark.parametrize("G", [1, 2, 4, 8])
@pytest.mark.parametrize("B", [6, 64])
def test_decode_attention_bit_identical(G, B):
    Hkv, Smax = 2, 512
    Hq = G * Hkv
    (kq, ki, kh), (vq, vi, vh) = _fp8_cache(B, Hkv, Smax, G * 100 + B)
    q = torch.randn(B, (Hq + 2 * Hkv) * D, device=DEV).bfloat16()
    pos = _positions(B, Smax, 1, B)
    nch = DK.attn_chunks(Smax)
    po, pm = torch.empty(B, Hq, nch, D, device=DEV), torch.empty(B, Hq, nch, 2, device=DEV)
    table = torch.randint(0, B, (B, nch), device=DEV, dtype=torch.int32)
    for t in (None, table):
        a = torch.empty(B, Hq * D, dtype=torch.bfloat16, device=DEV)
        b = torch.empty_like(a)
        DK.attention(q, kh, vh, pos, a, Hq, Hkv, D, po, pm, table=t)
        DK.attention(q, kq, vq, pos, b, Hq, Hkv, D, po, pm, table=t, kinv=ki, vinv=vi)
        assert torch.isfinite(a.float()).all()
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("G", [1, 2, 4, 8])
@pytest.mark.parametrize("n", list(range(1, 9)))
def test_verify_attention_bit_identical(G, n):
    Hkv, Smax, B = 2, 384, 8 if n % 2 else 64
    Hq = G * Hkv
    (kq, ki, kh), (vq, vi, vh) = _fp8_cache(B, Hkv, Smax, G * 10 + n)
    q = torch.randn(n * B, (Hq + 2 * Hkv) * D, device=DEV).bfloat16()
    pos = _positions(B, Smax, n, n)
    nsp = DK.verify_splits(Smax)
    po, pm = torch.empty(n * B, Hq, nsp, D, device=DEV), torch.empty(n * B, Hq, nsp, 2, device=DEV)
    a = torch.empty(n * B, Hq * D, dtype=torch.bfloat16, device=DEV)
    b = torch.empty_like(a)
    DK.verify_attention(q, kh, vh, pos, a, Hq, Hkv, D, n, po, pm)
    DK.verify_attention(q, kq, vq, pos, b, Hq, Hkv, D, n, po, pm, kinv=ki, vinv=vi)
    assert torch.isfinite(a.float()).all()
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


@pytest.mark.parametrize("p", [0, 5, 128, 300, 511])
def test_beam_reorder(p):
    L, nb, B, Hkv, Smax = 2, 4, 3, 2, 512
    rows = nb * B
    g = torch.Generator(device=DEV).manual_seed(p)
    kv = torch.randint(0, 126, (L, 2, rows, Hkv, Smax, D), device=DEV, generator=g, dtype=torch.uint8).view(E4M3)
    inv = torch.rand(L, 2, rows, Hkv, Smax, device=DEV, generator=g)
    table = torch.arange(rows, dtype=torch.int32, device=DEV)[:, None].repeat(1, Smax // 128).contiguous()
    pos = torch.full((rows,), p, dtype=torch.int32, device=DEV)
    ref_kv, ref_inv = kv.clone(), inv.clone()
    for step in range(3):                              # a few steps: tables compose
        parent = (torch.randint(0, nb, (rows,), device=DEV, generator=g) + torch.arange(B, device=DEV).repeat_interleave(nb) * nb)
        parent = parent.int()
        DK.beam_reorder(kv, table, parent, pos, nb, inv=inv)
        DK.beam_reorder_reference(ref_kv, parent, ref_inv)
    for l in range(L):
        for s in range(2):
            got = DK.gather_chunks(kv[l, s].view(torch.uint8), table)[:, :, :p]
            assert torch.equal(got, ref_kv[l, s].view(torch.uint8)[:, :, :p])
            goti = DK.gather_chunks(inv[l, s][..., None], table)[:, :, :p, 0]
            assert torch.equal(goti, ref_inv[l, s][:, :, :p])


# ------------------------------------------------------------------------------------------------ end to end
_M = {}


def _model():
    if "m" not in _M:
        cfg = LlamaConfig.from_pretrained("60m")
        _M["m"] = LlamaForCausalLM(cfg, device=DEV, precision="bf16-mixed", seed=3)
    return _M["m"]


def _ids(V, B, P, seed):
    ids = torch.randint(3, V, (B, P), generator=torch.Generator().manual_seed(seed))
    ids[:, P // 2:P // 2 + 12] = ids[:, 4:16]          # something for prompt lookup to find
    mask = torch.ones_like(ids)
    mask[1, :5] = 0
    return ids.to(DEV), mask.to(DEV)


MODES = {"greedy": {}, "sample": {"do_sample": True, "top_k": 50, "top_p": 0.9, "temperature": 0.9, "seed": 5},
         "processors": {"repetition_penalty": 1.2, "no_repeat_ngram_size": 3, "min_new_tokens": 4, "eos_token_id": [7]},
         "beam": {"num_beams": 3, "num_return_sequences": 2, "return_dict_in_generate": True},
         "lookup": {"prompt_lookup_num_tokens": 4},
         "assisted": {"num_assistant_tokens": 3}}


@pytest.mark.parametrize("fp8_weights", [False, True])
@pytest.mark.parametrize("mode", list(MODES))
def test_generate_equals_oracle(mode, fp8_weights, monkeypatch):
    m = _model()
    ids, mask = _ids(m.config.vocab_size, 4, 140, 1)
    kw = dict(MODES[mode], fp8_weights=fp8_weights)
    kw.setdefault("eos_token_id", [])
    if mode == "assisted":
        kw["assistant_model"] = m
    graph = m.generate(ids, attention_mask=mask, max_new_tokens=24, fp8_kv_cache=True, **kw)
    monkeypatch.setenv("ODB_CUDA_GRAPH", "0")
    eager = m.generate(ids, attention_mask=mask, max_new_tokens=24, fp8_kv_cache=True, **kw)
    ref = oracle_generate(m, ids, attention_mask=mask, max_new_tokens=24, **kw)
    for got in (graph, eager):
        if mode == "beam":
            assert torch.equal(got.sequences, ref.sequences)
            assert torch.equal(got.sequences_scores, ref.sequences_scores)
        else:
            assert torch.equal(got, ref)


def test_toggle_memory_and_recapture():
    m = _model()
    cfg = m.config
    ids, mask = _ids(cfg.vocab_size, 8, 100, 2)
    plain = m.generate(ids, attention_mask=mask, max_new_tokens=20, eos_token_id=[])
    st = m.engine.decode_state
    bf16_bytes = st.kv.numel() * st.kv.element_size()
    fp8 = m.generate(ids, attention_mask=mask, max_new_tokens=20, eos_token_id=[], fp8_kv_cache=True)
    s8 = m.engine.decode_state
    assert s8 is not st and s8.graph is not None and s8.kv.dtype == E4M3
    fp8_bytes = s8.kv.numel() * s8.kv.element_size() + s8.kv_inv.numel() * s8.kv_inv.element_size()
    assert fp8_bytes <= 0.54 * bf16_bytes
    assert torch.equal(m.generate(ids, attention_mask=mask, max_new_tokens=20, eos_token_id=[]), plain)
    assert not m.engine.decode_state.fp8_kv and m.engine.decode_state.graph is not None
    assert torch.equal(m.generate(ids, attention_mask=mask, max_new_tokens=20, eos_token_id=[], fp8_kv_cache=True), fp8)


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
m.generate(ids, max_new_tokens=4, eos_token_id=[], fp8_kv_cache=True)
st = m.engine.decode_state
from torch.profiler import ProfilerActivity, profile
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    step(m, st, graph=False)
    torch.cuda.synchronize()
print(json.dumps({"gpu": [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]}))
"""


def test_decode_step_runs_only_our_kernels():
    ours = set()
    for src in CSRC.glob("*.cu"):
        ours |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(", src.read_text()))
    res = subprocess.run([sys.executable, "-c", _PROFILE_STEP], capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    gpu = json.loads(res.stdout.strip().splitlines()[-1])["gpu"]
    assert gpu
    foreign = [n for n in gpu if not any(re.search(rf"\b{k}\b", n) for k in ours)]
    assert not foreign, foreign
    fp8 = [n for n in gpu if "unsigned char" in n]
    assert sum("rope_append_kernel" in n for n in fp8) == 2 and sum("decode_attn_kernel" in n for n in fp8) == 2
