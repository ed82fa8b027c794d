"""Multi-sample generation on the sm_90a decode kernels (H100).

- Grouped attention: ``attention_grouped`` (one load per shared chunk) equals ``attention`` through the same chunk table
  bit for bit, in the output and in the partials before the combine: G 1, 2, 4, 8; bf16 and FP8 caches; 1 to 64 siblings;
  prompt lengths 1 .. 2047 around the chunk edges; siblings at different positions; chunks shared by some siblings and
  not by others; the sibling split the launcher picks and every forced split.
- Fork: the caches of the B * n rows read through the forked table hold the bytes (and FP8 inv) the repeated-prompt
  prefill writes, up to every row's length.
- End to end: ``generate(do_sample=True, num_return_sequences=n)`` gives exactly the tokens of the repeated-prompt
  program (60m and 1b shapes, random weights, and the golden 2m), graph and eager, with the warpers, the logits processors,
  EOS, FP8 weights and the FP8 cache; the first-token logits after the prefill are the same bits.
- A forked decode step launches only the project's kernels; plain -> forked -> plain generation recaptures.

The module's name sorts it after the suite's in-process profiler tests.  On H100 hosts the profiler's GPU timestamps drift
from the host clock by about 0.17 ms per second after its first session and kernels outside the host window are dropped,
so a minute of extra GPU tests between two in-process profiler sessions leaves the later one without kernels."""
import gc
import json
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
from opendiloco_b200.ops.fp8 import E4M3

pytestmark = pytest.mark.gpu
DEV = "cuda"
D = 64
ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "opendiloco_b200" / "csrc"


# ------------------------------------------------------------------------------------------------ grouped attention
def _cache(rows, Hkv, Smax, fp8, g):
    """Random K and V [rows, Hkv, Smax, D] (bf16), or their e4m3 bytes and inv (FP8)."""
    out = []
    for _ in range(2):
        x = (torch.randn(rows, Hkv, Smax, D, device=DEV, generator=g) * 2).to(torch.bfloat16)
        if not fp8:
            out += [x, None]
            continue
        q, inv = FW.quantize_rows_ref(x.view(-1, D))
        out += [q.view(rows, Hkv, Smax, D), inv.view(rows, Hkv, Smax)]
    return out


def _group_case(P, n, Smax, lens, seed):
    """Positions and chunk table of P prompts of n siblings after a fork at lens[p] and j % 3 further tokens for sibling j:
    complete prompt chunks point at row p * n, except chunk 0 of every fourth sibling (its own copy); later chunks are the
    row's own."""
    rows, nch = P * n, Smax // 128
    pos = torch.empty(rows, dtype=torch.int32)
    table = torch.empty(rows, nch, dtype=torch.int32)
    for p in range(P):
        for j in range(n):
            r = p * n + j
            pos[r] = min(lens[p] - 1 + j % 3, Smax - 1)
            for c in range(nch):
                table[r, c] = p * n if c < lens[p] // 128 and not (j % 4 == 3 and c == 0) else r
    return pos.to(DEV), table.to(DEV)


CASES = [  # P, n, Smax, prompt lengths
    (1, 8, 2048, [2047]),
    (3, 2, 2048, [1000, 2047, 128]),
    (2, 17, 1152, [1000, 129]),
    (8, 3, 256, [1, 127, 128, 129, 1, 127, 128, 129]),
    (4, 64, 384, [128, 1, 129, 255]),
    (5, 1, 512, [300, 1, 128, 511, 2]),
]


@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("G", [1, 2, 4, 8])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_grouped_attention_bitwise(case, G, fp8):
    P, n, Smax, lens = CASES[case]
    Hkv = 2
    Hq = G * Hkv
    rows = P * n
    g = torch.Generator(device=DEV).manual_seed(100 + case * 8 + G)
    kc, kinv, vc, vinv = _cache(rows, Hkv, Smax, fp8, g)
    pos, table = _group_case(P, n, Smax, lens, case)
    q = torch.randn(rows, (Hq + 2 * Hkv) * D, device=DEV, generator=g).to(torch.bfloat16)
    nch = DK.attn_chunks(Smax)
    parts = lambda: (torch.zeros(rows, Hq, nch, D, device=DEV), torch.zeros(rows, Hq, nch, 2, device=DEV))  # noqa: E731
    po, pm = parts()
    ref = torch.empty(rows, Hq * D, dtype=torch.bfloat16, device=DEV)
    DK.attention(q, kc, vc, pos, ref, Hq, Hkv, D, po, pm, table=table, kinv=kinv, vinv=vinv)
    auto = DK.attn_group_splits(rows, n, Hq, Hkv, Smax, fp8)
    assert auto == 0 if (fp8 and G == 1) else 1 <= auto <= n
    for splits in sorted({0, 1, 2, 3, n} - {s for s in (2, 3) if s > n}):
        go, gm = parts()
        out = torch.full_like(ref, float("nan"))
        DK.attention_grouped(q, kc, vc, pos, out, Hq, Hkv, D, n, go, gm, table=table, kinv=kinv, vinv=vinv, splits=splits)
        torch.cuda.synchronize()
        assert torch.equal(go, po), splits
        assert torch.equal(gm, pm), splits
        assert torch.equal(out, ref), splits


# ------------------------------------------------------------------------------------------------ fork
@pytest.mark.parametrize("fp8", [False, True])
def test_fork_equals_repeated_prefill(fp8):
    L, Hq, Hkv, Smax, n = 2, 4, 2, 1152, 5
    lens = torch.tensor([1, 127, 128, 129, 1000, 1024], dtype=torch.int32, device=DEV)
    B, Sp = lens.numel(), 1024
    g = torch.Generator(device=DEV).manual_seed(7)
    qkv = torch.randn(L, B * Sp, (Hq + 2 * Hkv) * D, device=DEV, generator=g).to(torch.bfloat16)
    rows = B * n
    dt = E4M3 if fp8 else torch.bfloat16
    kv = torch.zeros(L, 2, rows, Hkv, Smax, D, dtype=dt, device=DEV)
    ref = torch.zeros_like(kv)
    inv = torch.zeros(L, 2, rows, Hkv, Smax, device=DEV) if fp8 else None
    ref_inv = torch.zeros_like(inv) if fp8 else None
    table = torch.full((rows, Smax // 128), -1, dtype=torch.int32, device=DEV)
    rep = qkv.view(L, B, Sp, -1).repeat_interleave(n, dim=1).reshape(L, rows * Sp, -1)
    for l in range(L):
        iv = lambda t, s: t[l, s] if t is not None else None  # noqa: E731
        DK.kv_fill(qkv[l], lens, kv[l, 0], kv[l, 1], B, Sp, Hq, Hkv, D, row_stride=n, kinv=iv(inv, 0), vinv=iv(inv, 1))
        DK.kv_fill(rep[l], lens.repeat_interleave(n), ref[l, 0], ref[l, 1], rows, Sp, Hq, Hkv, D, kinv=iv(ref_inv, 0),
                   vinv=iv(ref_inv, 1))
    DK.fork(kv, table, lens, n, inv=inv)
    torch.cuda.synchronize()
    for r in range(rows):
        p, j = divmod(r, n)
        c = int(lens[p]) // 128
        want = [p * n if (j > 0 and cc < c) else r for cc in range(Smax // 128)]
        assert table[r].tolist() == want
    for l in range(L):
        for s in range(2):
            raw = (lambda t: t.view(torch.uint8)) if fp8 else (lambda t: t)
            got = DK.gather_chunks(raw(kv[l, s]), table)
            for r in range(rows):
                m = int(lens[r // n])
                assert torch.equal(got[r, :, :m], raw(ref[l, s])[r, :, :m])
                if fp8:
                    gi = DK.gather_chunks(inv[l, s][..., None], table)[r, :, :m, 0]
                    assert torch.equal(gi, ref_inv[l, s][r, :, :m])


# ------------------------------------------------------------------------------------------------ end to end
_M = {}


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    """The models of this module (1b included), their decode states and captured graphs are freed when it ends."""
    yield
    _M.clear()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _model(name):
    if name not in _M:
        if name == "2m":
            _M[name] = LlamaForCausalLM.from_pretrained(str(ROOT / "tests" / "golden" / "llama-2m-fresh"), device=DEV,
                                                        precision="bf16-mixed")
        else:
            _M[name] = LlamaForCausalLM(LlamaConfig.from_pretrained(name), device=DEV, precision="bf16-mixed", seed=5)
    return _M[name]


def _ids(V, B, P, seed):
    ids = torch.randint(3, V, (B, P), generator=torch.Generator().manual_seed(seed))
    mask = torch.ones_like(ids)
    if B > 1:
        mask[1, :P - 128] = 0                             # a prompt of exactly 128 tokens
        mask[B - 1, :7] = 0
    return ids.to(DEV), mask.to(DEV)


def _first_logits(m, ids, mask, n, **kw):
    """The logits rows after the prefill of the forked and of the repeated program."""
    out = []
    for group in (n, 1):
        m.generate(ids if group > 1 else ids.repeat_interleave(n, 0), attention_mask=mask if group > 1 else mask.repeat_interleave(n, 0),
                   max_new_tokens=1, num_return_sequences=group, do_sample=True, eos_token_id=[], **kw)
        out.append(m.engine.decode_state.logits.clone())
    return out


SAMPLING = {"t1": dict(temperature=1.0, top_k=0),
            "t07": dict(temperature=0.7, top_k=40, top_p=0.9),
            "processors": dict(temperature=0.8, repetition_penalty=1.3, no_repeat_ngram_size=2, min_new_tokens=5),
            "eos": dict(temperature=1.0, top_k=8),
            "fp8_weights": dict(temperature=0.7, top_p=0.95, fp8_weights=True),
            "fp8_kv": dict(temperature=0.7, top_p=0.95, fp8_kv_cache=True),
            "fp8_both": dict(temperature=1.0, top_k=50, fp8_weights=True, fp8_kv_cache=True, repetition_penalty=1.1)}

# every mode once at 60m, the (n, B) pairs cycling through (2, 4), (8, 1), (16, 4); the 1b and 2m shapes on a few modes
NEW = 40
E2E = [("60m", mode, n, B) for mode in SAMPLING for n, B in ((2, 4), (8, 1), (16, 4))] + \
      [("1b", mode, 8, B) for mode in ("t07", "fp8_kv") for B in (1, 4)] + [("2m", mode, 8, 4) for mode in ("t1", "processors")]


@pytest.mark.parametrize("name,mode,n,B", E2E)
def test_generate_equals_repeated_program(name, mode, n, B, monkeypatch):
    m = _model(name)
    V = m.config.vocab_size
    ids, mask = _ids(V, B, 200, n * 10 + B)
    kw = dict(SAMPLING[mode], seed=11, max_new_tokens=NEW, do_sample=True)
    fl = {k: kw[k] for k in ("fp8_weights", "fp8_kv_cache") if k in kw}
    got_logits, ref_logits = _first_logits(m, ids, mask, n, **fl)
    assert torch.equal(got_logits, ref_logits)
    if mode == "eos":                                     # EOS ids hit early: the two most likely first tokens of row 0
        kw["eos_token_id"] = ref_logits[0].float().topk(2).indices.tolist()
    kw.setdefault("eos_token_id", [])
    rep = dict(attention_mask=mask.repeat_interleave(n, 0), **kw)
    ref = m.generate(ids.repeat_interleave(n, 0), **rep)
    graph = m.generate(ids, attention_mask=mask, num_return_sequences=n, **kw)
    monkeypatch.setenv("ODB_CUDA_GRAPH", "0")
    eager = m.generate(ids, attention_mask=mask, num_return_sequences=n, **kw)
    assert graph.shape == (B * n, ids.shape[1] + NEW)
    assert torch.equal(graph, ref)
    assert torch.equal(eager, ref)
    if mode == "eos":
        assert bool(torch.isin(ref[:, ids.shape[1]:-1], torch.tensor(kw["eos_token_id"], device=DEV)).any())
    if name != "2m":
        assert m.engine.decode_state.table is not None and m.engine.decode_state.group == n


def test_toggle_plain_forked_plain():
    m = _model("60m")
    ids, mask = _ids(m.config.vocab_size, 4, 150, 9)
    kw = dict(max_new_tokens=24, do_sample=True, seed=3, eos_token_id=[])
    plain = m.generate(ids, attention_mask=mask, **kw)
    st_plain = m.engine.decode_state
    assert st_plain.table is None and st_plain.graph is not None
    forked = m.generate(ids, attention_mask=mask, num_return_sequences=4, **kw)
    st_forked = m.engine.decode_state
    assert st_forked is not st_plain and st_forked.group == 4 and st_forked.graph is not None
    again = m.generate(ids, attention_mask=mask, **kw)
    assert m.engine.decode_state.group == 1 and m.engine.decode_state.table is None
    assert torch.equal(again, plain)
    assert torch.equal(forked, m.generate(ids.repeat_interleave(4, 0), attention_mask=mask.repeat_interleave(4, 0), **kw))


_PROFILE_STEP = r"""
import json, os, sys
import torch
sys.path.insert(0, os.getcwd())
from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.generation import step
from opendiloco_b200.models.llama import LlamaForCausalLM
cfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=2, num_attention_heads=16, vocab_size=32000)
m = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=1)
ids = torch.randint(3, 32000, (2, 300), device="cuda")
from torch.profiler import ProfilerActivity, profile
res = {}
for fp8_kv in (False, True):
    m.generate(ids, max_new_tokens=4, eos_token_id=[], do_sample=True, num_return_sequences=8, fp8_kv_cache=fp8_kv)
    st = m.engine.decode_state
    assert st.group == 8 and st.table is not None
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        step(m, st, graph=False)
        torch.cuda.synchronize()
    res[str(int(fp8_kv))] = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
print(json.dumps(res))
"""


def test_forked_step_runs_only_our_kernels():
    """bf16 and FP8 caches, profiled in one fresh process."""
    ours = set()
    for src in CSRC.glob("*.cu"):
        ours |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(", src.read_text()))
    res = subprocess.run([sys.executable, "-c", _PROFILE_STEP], capture_output=True, text=True, cwd=ROOT, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    out = json.loads(res.stdout.strip().splitlines()[-1])
    for fp8_kv in (False, True):
        gpu = out[str(int(fp8_kv))]
        assert gpu
        foreign = [n for n in gpu if not any(re.search(rf"\b{k}\b", n) for k in ours)]
        assert not foreign, foreign
        # 16 heads of 16 kv heads: the FP8 cache at G = 1 runs decode_attn_kernel through the table (attn_group_splits 0)
        grouped, plain = (sum(bool(re.search(rf"\b{k}\b", n)) for n in gpu) for k in ("decode_attn_group_kernel", "decode_attn_kernel"))
        assert (grouped, plain) == ((0, 2) if fp8_kv else (2, 0))
