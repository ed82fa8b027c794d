"""FP8 KV cache (``generate(fp8_kv_cache=True)``) on the PyTorch reference path (CPU, head_dim 32 presets).

The oracle is today's bf16-cache program with every cache write followed by replacing the written rows with their
dequantised values ``dequantize_rows(*quantize_rows_ref(rows))``: a test-local wrapper around the three cache writers
(``oracle_writers``).  Every generation mode must give exactly its tokens.  Also covered: the cache layout the writers
produce (ragged lengths, the beam prefill's row stride, the verify writes at pos + j), zero / exactly-448 / NaN rows,
the readers and the beam reorder on the FP8 cache, the error, the unchanged default allocation and the CLI flag."""
import contextlib
import os
import subprocess
import sys

import pytest
import torch

from opendiloco_b200.models import generation as GEN
from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import decode as DK
from opendiloco_b200.ops import fp8w as FW
from opendiloco_b200.ops.fp8 import E4M3

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GEN_SCRIPT = os.path.join(ROOT, "scripts", "generate.py")


def hat(x: torch.Tensor) -> torch.Tensor:
    """x [..., D] with every row replaced by its quantised-dequantised value Ĉ."""
    q, inv = FW.quantize_rows_ref(x.reshape(-1, x.shape[-1]))
    return FW.dequantize_rows(q, inv, x.dtype).view(x.shape)


@contextlib.contextmanager
def oracle_writers(model):
    """Wrap the bf16 cache writers of ops.decode so the rows they write are replaced by Ĉ.  The caches of an assisted
    generation's draft (``engine.assisted_state.draft``) are left alone: only the target's cache is FP8."""
    orig = DK.rope_append, DK.rope_append_multi, DK.kv_fill

    def target(kc):
        ast = model.engine.assisted_state
        return not (ast is not None and ast.draft is not None
                    and kc.untyped_storage().data_ptr() == ast.draft.kv.untyped_storage().data_ptr())

    def rope_append(qkv, cos, sin, pos, kc, vc, Hq, Hkv, D, kinv=None, vinv=None):
        assert kinv is None
        orig[0](qkv, cos, sin, pos, kc, vc, Hq, Hkv, D)
        if target(kc):
            rows, p = torch.arange(kc.shape[0], device=kc.device), pos.long().to(kc.device)
            for c in (kc, vc):
                c[rows, :, p] = hat(c[rows, :, p])

    def rope_append_multi(qkv, cos, sin, pos, kc, vc, Hq, Hkv, D, n, kinv=None, vinv=None):
        assert kinv is None
        orig[1](qkv, cos, sin, pos, kc, vc, Hq, Hkv, D, n)
        if target(kc):
            B = qkv.shape[0] // n
            rows = torch.arange(B, device=kc.device).repeat(n)
            p = (pos.long().to(kc.device)[None, :] + torch.arange(n, device=kc.device)[:, None]).reshape(-1)
            for c in (kc, vc):
                c[rows, :, p] = hat(c[rows, :, p])

    def kv_fill(qkv, lens, kc, vc, B, Sp, Hq, Hkv, D, row_stride=1, kinv=None, vinv=None):
        assert kinv is None
        orig[2](qkv, lens, kc, vc, B, Sp, Hq, Hkv, D, row_stride=row_stride)
        if target(kc):
            n = min(Sp, kc.shape[2])
            keep = (torch.arange(n, device=kc.device)[None, :] < lens.long().to(kc.device)[:, None])[:, None, :, None]
            for c in (kc, vc):
                d = c[::row_stride]
                d[:, :, :n] = torch.where(keep, hat(d[:, :, :n]), d[:, :, :n])

    DK.rope_append, DK.rope_append_multi, DK.kv_fill = rope_append, rope_append_multi, kv_fill
    try:
        yield
    finally:
        DK.rope_append, DK.rope_append_multi, DK.kv_fill = orig


def oracle_generate(model, *args, **kw):
    with oracle_writers(model):
        return model.generate(*args, **kw)


def _prompts(V, B=3, P=10, seed=0):
    ids = torch.randint(3, V, (B, P), generator=torch.Generator().manual_seed(seed))
    mask = torch.ones_like(ids)
    mask[1, :4] = 0
    return ids.masked_fill(mask == 0, 0), mask


@pytest.fixture(scope="module")
def model(ref_model_dir):
    return LlamaForCausalLM.from_pretrained(ref_model_dir, precision="32-true")


MODES = {"greedy": {}, "sample": {"do_sample": True, "top_k": 20, "top_p": 0.9, "temperature": 0.8, "seed": 11},
         "beam": {"num_beams": 3, "num_return_sequences": 2, "return_dict_in_generate": True},
         "beam_eos": {"num_beams": 2, "eos_token_id": [7, 11], "early_stopping": True, "return_dict_in_generate": True},
         "lookup": {"prompt_lookup_num_tokens": 3},
         "processors": {"repetition_penalty": 1.3, "no_repeat_ngram_size": 2, "min_new_tokens": 5},
         "eos": {"eos_token_id": [5, 9, 13, 17, 21], "pad_token_id": 1},
         "assisted": {"num_assistant_tokens": 3},
         "fp8_weights": {"fp8_weights": True},
         "beam_fp8_weights": {"num_beams": 2, "return_dict_in_generate": True, "fp8_weights": True},
         "assisted_fp8_weights": {"num_assistant_tokens": 2, "fp8_weights": True}}


def _same(got, ref):
    if isinstance(got, GEN.GenerateOutput):
        assert torch.equal(got.sequences, ref.sequences)
        if ref.sequences_scores is not None:
            assert torch.equal(got.sequences_scores, ref.sequences_scores)
    else:
        assert torch.equal(got, ref)


@pytest.mark.parametrize("mode", list(MODES))
def test_generate_equals_oracle(model, mode):
    ids, mask = _prompts(model.config.vocab_size)
    kw = dict(MODES[mode])
    if mode.startswith("assisted"):
        kw["assistant_model"] = model                   # the model drafts for itself: its draft cache stays bf16
    got = model.generate(ids, attention_mask=mask, max_new_tokens=12, fp8_kv_cache=True, **kw)
    ref = oracle_generate(model, ids, attention_mask=mask, max_new_tokens=12, **kw)
    _same(got, ref)


def test_fp8_cache_changes_the_program(model):
    """The oracle wrapper is not a no-op: the dequantised cache differs from the bf16 one."""
    ids, mask = _prompts(model.config.vocab_size, B=4, P=24, seed=5)
    model.generate(ids, attention_mask=mask, max_new_tokens=4)
    kv = model.engine.decode_state.kv.clone()
    oracle_generate(model, ids, attention_mask=mask, max_new_tokens=4)
    assert not torch.equal(model.engine.decode_state.kv, kv)


def test_14m_greedy_beam_lookup():
    cfg = LlamaConfig.from_pretrained("14m")
    cfg.vocab_size = 512
    m = LlamaForCausalLM(cfg, precision="32-true", seed=3)
    ids, mask = _prompts(cfg.vocab_size, B=2, P=9, seed=4)
    for kw in ({}, {"num_beams": 3, "return_dict_in_generate": True}, {"prompt_lookup_num_tokens": 2}):
        _same(m.generate(ids, attention_mask=mask, max_new_tokens=7, fp8_kv_cache=True, **kw),
              oracle_generate(m, ids, attention_mask=mask, max_new_tokens=7, **kw))


# ------------------------------------------------------------------------------------------------ state and layout
def test_state_layout_and_toggle(model):
    cfg = model.config
    ids, mask = _prompts(cfg.vocab_size)
    a = model.generate(ids, attention_mask=mask, max_new_tokens=6)
    st = model.engine.decode_state
    L, Hkv, D = cfg.num_hidden_layers, cfg.num_key_value_heads, cfg.head_dim
    assert st.kv.dtype == torch.float32 and st.kv_inv is None and not st.fp8_kv       # the default allocates today's cache
    assert st.kv.shape == (L, 2, 3, Hkv, st.Smax, D) and st.kinv == [None] * L
    model.generate(ids, attention_mask=mask, max_new_tokens=6, fp8_kv_cache=True)
    s8 = model.engine.decode_state
    assert s8 is not st and s8.fp8_kv and s8.kv.dtype == E4M3 and s8.kv_inv.dtype == torch.float32
    assert s8.kv.shape == (L, 2, 3, Hkv, s8.Smax, D) and s8.kv_inv.shape == (L, 2, 3, Hkv, s8.Smax)
    assert s8.kc[1].data_ptr() == s8.kv[1, 0].data_ptr() and s8.vinv[1].data_ptr() == s8.kv_inv[1, 1].data_ptr()
    # bytes per head-position: D e4m3 + 4 (inv) against 2 * D bf16
    assert (D + 4) / (2 * D) <= 0.57
    assert torch.equal(model.generate(ids, attention_mask=mask, max_new_tokens=6, fp8_kv_cache=False), a)
    assert not model.engine.decode_state.fp8_kv


@pytest.mark.parametrize("bad", [1, 0, "yes", None, 1.0])
def test_errors(model, bad):
    ids, _ = _prompts(model.config.vocab_size)
    with pytest.raises(ValueError, match="fp8_kv_cache"):
        model.generate(ids, max_new_tokens=2, fp8_kv_cache=bad)


def _cache(B, Hkv, Smax, D, fp8):
    if fp8:
        return (torch.zeros(B, Hkv, Smax, D, dtype=E4M3), torch.zeros(B, Hkv, Smax, D, dtype=E4M3),
                torch.zeros(B, Hkv, Smax), torch.zeros(B, Hkv, Smax))
    return torch.zeros(B, Hkv, Smax, D, dtype=torch.bfloat16), torch.zeros(B, Hkv, Smax, D, dtype=torch.bfloat16), None, None


def _rope_tables(n, D):
    ang = torch.arange(n)[:, None].float() * (10000.0 ** (-torch.arange(D // 2).float() * 2 / D))[None, :]
    return ang.cos(), ang.sin()


def _assert_quantised(kq, ki, kb, written):
    """The FP8 cache (bytes, inv) holds quantize_rows_ref of the bf16 cache kb in the written rows (bool [B, Smax]) and
    zeros elsewhere."""
    D = kb.shape[-1]
    w = written[:, None, :].expand(ki.shape)
    q, inv = FW.quantize_rows_ref(kb[w])
    assert torch.equal(kq.view(torch.uint8)[w], q.view(torch.uint8))
    torch.testing.assert_close(ki[w], inv, rtol=0, atol=0, equal_nan=True)
    assert (kq.view(torch.uint8)[~w] == 0).all() and (ki[~w] == 0).all()


def test_writers_layout():
    """rope_append at ragged positions, rope_append_multi at pos + j, kv_fill with ragged lens and a beam row stride:
    every written row holds the quantised bf16 row, every other row stays zero (bytes 0, inv 0)."""
    B, Hq, Hkv, D, Smax, n = 4, 4, 2, 32, 64, 3
    cos, sin = _rope_tables(Smax + 8, D)
    g = torch.Generator().manual_seed(0)
    qkv = (torch.randn(n * B, (Hq + 2 * Hkv) * D, generator=g) * 3).bfloat16()
    pos = torch.tensor([0, 5, 31, 60], dtype=torch.int32)
    for multi in (False, True):
        x = qkv if multi else qkv[:B]
        kb, vb, _, _ = _cache(B, Hkv, Smax, D, False)
        kq, vq, ki, vi = _cache(B, Hkv, Smax, D, True)
        a, b = x.clone(), x.clone()
        if multi:
            DK.rope_append_multi(a, cos, sin, pos, kb, vb, Hq, Hkv, D, n)
            DK.rope_append_multi(b, cos, sin, pos, kq, vq, Hq, Hkv, D, n, kinv=ki, vinv=vi)
        else:
            DK.rope_append(a, cos, sin, pos, kb, vb, Hq, Hkv, D)
            DK.rope_append(b, cos, sin, pos, kq, vq, Hq, Hkv, D, kinv=ki, vinv=vi)
        assert torch.equal(a, b)                                                    # the same rotated q
        want = torch.zeros(B, Smax, dtype=torch.bool)
        for j in range(n if multi else 1):
            want[torch.arange(B), pos.long() + j] = True
        _assert_quantised(kq, ki, kb, want)
        _assert_quantised(vq, vi, vb, want)
    # prefill: ragged lens, beam rows (row_stride 2: prompt b fills row 2b)
    Sp, lens = 8, torch.tensor([8, 3], dtype=torch.int32)
    x = (torch.randn(2 * Sp, (Hq + 2 * Hkv) * D, generator=g) * 0.01).bfloat16()
    kb, vb, _, _ = _cache(4, Hkv, Smax, D, False)
    kq, vq, ki, vi = _cache(4, Hkv, Smax, D, True)
    DK.kv_fill(x, lens, kb, vb, 2, Sp, Hq, Hkv, D, row_stride=2)
    DK.kv_fill(x, lens, kq, vq, 2, Sp, Hq, Hkv, D, row_stride=2, kinv=ki, vinv=vi)
    want = torch.zeros(4, Smax, dtype=torch.bool)
    want[0, :8], want[2, :3] = True, True
    _assert_quantised(kq, ki, kb, want)
    _assert_quantised(vq, vi, vb, want)


def test_special_rows():
    """A zero row (bytes 0, inv 1), a row with amax exactly 448 (scale 1), a NaN row and an inf row (NaN bytes, inv NaN)."""
    Hq, Hkv, D, Smax = 1, 1, 64, 8
    rows = torch.zeros(4, D)
    rows[1, 3], rows[1, 7] = 448.0, -3.0
    rows[2, 5] = float("nan")
    rows[3, 9] = float("inf")
    qkv = torch.zeros(4, (Hq + 2 * Hkv) * D, dtype=torch.bfloat16)
    qkv[:, Hq * D:(Hq + 1) * D] = rows.bfloat16()
    qkv[:, (Hq + 1) * D:] = rows.bfloat16()
    kq, vq, ki, vi = _cache(1, Hkv, Smax, D, True)
    DK.kv_fill(qkv, torch.tensor([4], dtype=torch.int32), kq, vq, 1, 4, Hq, Hkv, D, kinv=ki, vinv=vi)
    for c, inv in ((kq, ki), (vq, vi)):
        b = c.view(torch.uint8)[0, 0]
        assert (b[0] == 0).all() and inv[0, 0, 0] == 1.0
        assert inv[0, 0, 1] == 1.0 and c[0, 0, 1, 3].float() == 448.0 and c[0, 0, 1, 7].float() == -3.0
        assert (b[2] == 0x7F).all() and torch.isnan(inv[0, 0, 2])
        assert (b[3] == 0x7F).all() and torch.isnan(inv[0, 0, 3])


def test_readers_and_reorder():
    """attention / verify_attention / gather_chunks on the FP8 cache equal the bf16 references on Ĉ; beam_reorder moves
    bytes and inv together."""
    B, Hq, Hkv, D, Smax, n = 4, 4, 2, 32, 256, 3
    g = torch.Generator().manual_seed(1)
    kb = torch.randn(B, Hkv, Smax, D, generator=g).bfloat16()
    vb = torch.randn(B, Hkv, Smax, D, generator=g).bfloat16()
    (kq, ki), (vq, vi) = FW.quantize_rows_ref(kb.view(-1, D)), FW.quantize_rows_ref(vb.view(-1, D))
    kq, vq, ki, vi = kq.view(kb.shape), vq.view(vb.shape), ki.view(kb.shape[:-1]), vi.view(vb.shape[:-1])
    kh, vh = hat(kb), hat(vb)
    q = torch.randn(n * B, (Hq + 2 * Hkv) * D, generator=g).bfloat16()
    pos = torch.tensor([0, 127, 128, 200], dtype=torch.int32)
    table = torch.tensor([[0, 1], [1, 1], [2, 0], [3, 2]], dtype=torch.int32)
    for t in (None, table):
        a, b = torch.empty(B, Hq * D, dtype=torch.bfloat16), torch.empty(B, Hq * D, dtype=torch.bfloat16)
        DK.attention(q[:B], kh, vh, pos, a, Hq, Hkv, D, table=t)
        DK.attention(q[:B], kq, vq, pos, b, Hq, Hkv, D, table=t, kinv=ki, vinv=vi)
        assert torch.equal(a, b)
    a, b = torch.empty(n * B, Hq * D, dtype=torch.bfloat16), torch.empty(n * B, Hq * D, dtype=torch.bfloat16)
    DK.verify_attention(q, kh, vh, pos.clamp(max=Smax - n), a, Hq, Hkv, D, n)
    DK.verify_attention(q, kq, vq, pos.clamp(max=Smax - n), b, Hq, Hkv, D, n, kinv=ki, vinv=vi)
    assert torch.equal(a, b)
    assert torch.equal(DK.gather_chunks(kq, table, ki), DK.gather_chunks(kh, table))
    kv = torch.stack([kq, vq])[None].contiguous()
    inv = torch.stack([ki, vi])[None].contiguous()
    parent = torch.tensor([1, 1, 3, 2], dtype=torch.int32)
    kv2, inv2 = kv.clone(), inv.clone()
    DK.beam_reorder(kv2, None, parent, pos, 2, inv=inv2)
    idx = parent.long()
    assert torch.equal(kv2.view(torch.uint8), kv.view(torch.uint8)[:, :, idx]) and torch.equal(inv2, inv[:, :, idx])


def test_cli_flag(model, ref_model_dir):
    ids = [5, 9, 17, 33, 2]
    env = {**os.environ, "PYTHONPATH": ROOT + os.pathsep + os.environ.get("PYTHONPATH", "")}
    run = subprocess.run([sys.executable, GEN_SCRIPT, "--model", ref_model_dir, "--device", "cpu", "--prompt-ids", " ".join(map(str, ids)),
                          "--max-new-tokens", "8", "--eos-token-id", "-1", "--fp8-kv-cache"],
                         capture_output=True, text=True, env=env, cwd=ROOT)
    assert run.returncode == 0, run.stderr
    line = [x for x in run.stdout.splitlines() if x.startswith("ids:")][0]
    want = model.generate(torch.tensor([ids]), max_new_tokens=8, eos_token_id=-1, fp8_kv_cache=True)[0].tolist()
    assert [int(t) for t in line.split()[1:]] == want
    assert want == oracle_generate(model, torch.tensor([ids]), max_new_tokens=8, eos_token_id=-1)[0].tolist()
