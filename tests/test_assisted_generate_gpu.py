"""Assisted-generation kernels (csrc/decode_sm90.cu: multi-token RoPE+append, verify attention, acceptance) and
``generate(assistant_model=...)`` on an H100."""
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
from opendiloco_b200.ops import kernels as K

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "opendiloco_b200" / "csrc"


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm()).item()


@pytest.mark.parametrize("G", [1, 2, 4, 8])
@pytest.mark.parametrize("n", [1, 2, 5, 8])
def test_verify_attention_matches_fp32(G, n):
    D, Smax, Hkv = 64, 2048, 2
    Hq = G * Hkv
    positions = [0, 127 - n + 1, 127, 128, 129, 1000, Smax - n]   # slot-0 positions: chunk edges, the end of the cache
    positions = [max(p, 0) for p in positions]
    B = len(positions)
    g = torch.Generator(device="cuda").manual_seed(G * 10 + n)
    q = torch.randn(n * B, (Hq + 2 * Hkv) * D, device="cuda", generator=g).bfloat16()
    kc = torch.randn(B, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
    vc = torch.randn(B, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
    pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
    nsp = DK.verify_splits(Smax)
    part_o = torch.empty(n * B, Hq, nsp, D, device="cuda")
    part_ml = torch.empty(n * B, Hq, nsp, 2, device="cuda")
    out = torch.empty(n * B, Hq * D, dtype=torch.bfloat16, device="cuda")
    DK.verify_attention(q, kc, vc, pos, out, Hq, Hkv, D, n, part_o, part_ml)
    ref = torch.empty(n * B, Hq * D, dtype=torch.float32, device="cuda")
    DK.verify_attention(q.float(), kc.float(), vc.float(), pos, ref, Hq, Hkv, D, n)     # fp32: the PyTorch reference
    for j in range(n):
        for b, p in enumerate(positions):
            r = _rel(out[j * B + b], ref[j * B + b])
            assert r < 5e-3, (G, n, j, p, r)


@pytest.mark.parametrize("n", [1, 3, 8])
def test_rope_append_multi_matches_single_token_kernel(n):
    Hq, Hkv, D, Smax = 8, 2, 64, 512
    positions = [0, 5, 127 - n + 1, 128, 300, Smax - n]
    B = len(positions)
    g = torch.Generator(device="cuda").manual_seed(n)
    qkv = torch.randn(n * B, (Hq + 2 * Hkv) * D, device="cuda", generator=g).bfloat16()
    kc = torch.randn(B, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
    vc = torch.randn(B, Hkv, Smax, D, device="cuda", generator=g).bfloat16()
    cos, sin = K.rope_tables(Smax, D, 10000.0, "cuda")
    pos = torch.tensor(positions, dtype=torch.int32, device="cuda")
    # the single-token kernel, once per slot, is the exact reference
    q1, k1, v1 = qkv.clone(), kc.clone(), vc.clone()
    for j in range(n):
        DK.rope_append(q1[j * B:(j + 1) * B], cos, sin, pos + j, k1, v1, Hq, Hkv, D)
    # and the PyTorch reference agrees to one bf16 rounding
    qr, kr, vr = qkv.cpu(), kc.cpu(), vc.cpu()
    DK.rope_append_multi(qr, cos.cpu(), sin.cpu(), pos.cpu(), kr, vr, Hq, Hkv, D, n)
    DK.rope_append_multi(qkv, cos, sin, pos, kc, vc, Hq, Hkv, D, n)
    assert torch.equal(qkv, q1) and torch.equal(kc, k1) and torch.equal(vc, v1)
    assert _rel(qkv[:, : Hq * D], qr[:, : Hq * D].cuda()) < 4e-3
    assert _rel(kc, kr.cuda()) < 4e-3 and torch.equal(vc, vr.cuda())


def _accept_inputs(V, K, B, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    plog = (3 * torch.randn((K + 1) * B, V, device="cuda", generator=g)).bfloat16()
    qlog = (3 * torch.randn(K * B, V, device="cuda", generator=g)).bfloat16()
    return plog, qlog


def _run_accept(plog, qlog, tok, ctl, pos, gen, fin, max_new, out_w):
    B = pos.shape[0]
    ictl, fctl = ctl
    st = dict(tok=tok.clone(), pos=pos.clone(), gen=gen.clone(), fin=fin.clone(), dpos=torch.zeros_like(pos),
              out=torch.zeros(B, out_w, dtype=torch.int64, device=pos.device),
              stats=torch.zeros(B, 2, dtype=torch.int64, device=pos.device))
    DK.accept(plog, qlog, ictl, fctl, st["tok"], st["pos"], st["gen"], st["fin"], st["out"], max_new, st["dpos"], st["stats"])
    return st


def test_accept_greedy_matches_reference():
    V, K, B = 32000, 4, 64
    plog, qlog = _accept_inputs(V, K, B, 1)
    am = plog.float().view(K + 1, B, V).argmax(dim=-1)
    # proposals: the target argmax, with a wrong token planted at a row-dependent slot (slot K+1: none)
    tok = torch.zeros(K + 1, B, dtype=torch.int64, device="cuda")
    tok[1:] = am[:K]
    for b in range(B):
        s = b % (K + 2)
        if s < K:
            tok[1 + s, b] = (am[s, b] + 1) % V
    eos = int(am[1, 3])                                  # row 3 emits an EOS inside its block
    ctl = DK.make_controls(False, 1.0, 0, 1.0, 0, 0, [eos], "cuda")
    pos = torch.randint(5, 100, (B,), dtype=torch.int32, device="cuda")
    gen = torch.randint(1, 10, (B,), dtype=torch.int32, device="cuda")
    gen[7] = 11                                          # row 7 reaches max_new inside its block
    fin = torch.zeros(B, dtype=torch.int32, device="cuda")
    fin[9] = 1
    got = _run_accept(plog, qlog, tok.view(-1), ctl, pos, gen, fin, 12, 16)
    ref = _run_accept(plog.cpu(), qlog.cpu(), tok.view(-1).cpu(), [c.cpu() for c in ctl], pos.cpu(), gen.cpu(), fin.cpu(), 12, 16)
    for k in got:
        assert torch.equal(got[k].cpu(), ref[k]), k
    assert int(got["fin"][3]) == 1 and int(got["fin"][7]) == 1 and int(got["gen"][7]) == 12


def test_accept_sampling_chi_square_and_seed():
    scipy_stats = pytest.importorskip("scipy.stats")
    V, K, rows = 64, 2, 100_000
    g = torch.Generator().manual_seed(5)
    # distinct bf16 logits (no ties at the top-k / top-p edge); the draft favours what the target's warpers remove
    p_logits = torch.stack([torch.randperm(V, generator=g) * 0.08 for _ in range(K + 1)]).bfloat16()
    q_logits = (-p_logits[:K].float() + torch.randperm(V, generator=g)[None] * 0.01).bfloat16()
    for temperature, top_k, top_p in ((1.0, 0, 1.0), (0.7, 20, 1.0), (1.2, 0, 0.6), (0.9, 12, 0.8)):
        qw = torch.softmax(DK.warp_logits(q_logits.float(), temperature, top_k, top_p), dim=-1)
        tok = torch.zeros(K + 1, rows, dtype=torch.int64)
        tok[1:] = torch.stack([torch.multinomial(qw[i], rows, replacement=True, generator=g) for i in range(K)])
        ctl = DK.make_controls(True, temperature, top_k, top_p, 1234, 0, [], "cuda")
        plog = p_logits.cuda()[:, None].expand(K + 1, rows, V).reshape(-1, V)
        qlog = q_logits.cuda()[:, None].expand(K, rows, V).reshape(-1, V)
        z = torch.zeros(rows, dtype=torch.int32, device="cuda")
        a = _run_accept(plog, qlog, tok.view(-1).cuda(), ctl, z, z + 1, z, 16, 16)
        b = _run_accept(plog, qlog, tok.view(-1).cuda(), ctl, z, z + 1, z, 16, 16)
        for k in a:
            assert torch.equal(a[k], b[k]), k
        first = a["out"][:, 1].cpu()
        p1 = torch.softmax(DK.warp_logits(p_logits[:1].double(), temperature, top_k, top_p), dim=-1)[0]
        counts = torch.bincount(first, minlength=V).double()
        assert float(counts[p1 == 0].sum()) == 0
        keep = p1 > 0
        stat, pval = scipy_stats.chisquare(counts[keep].numpy(), (p1[keep] * rows).numpy())
        print("chi-square", (temperature, top_k, top_p), stat, pval, "acceptance", float(a["stats"][:, 1].sum()) / (K * rows))
        assert pval > 1e-3


def _pair():
    tcfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=4, num_attention_heads=16, vocab_size=32000)
    dcfg = LlamaConfig.from_pretrained("60m")
    return (LlamaForCausalLM(tcfg, device="cuda", precision="bf16-mixed", seed=1),
            LlamaForCausalLM(dcfg, device="cuda", precision="bf16-mixed", seed=2))


def _first_gap_index(model, seq, P):
    """Per row: the first new-token index whose plain-greedy top-2 logits differ by < 0.05 (or the length)."""
    with torch.no_grad():
        logits = model(seq).logits.float()              # [B, S, V]
    top2 = logits[:, P - 1:-1].topk(2, dim=-1).values
    close = (top2[..., 0] - top2[..., 1]) < 0.05
    n = seq.shape[1] - P
    return [int(torch.nonzero(close[b])[0]) if bool(close[b].any()) else n for b in range(seq.shape[0])]


@pytest.mark.parametrize("graph", ["1", "0"])
def test_greedy_end_to_end(graph, monkeypatch):
    monkeypatch.setenv("ODB_CUDA_GRAPH", graph)
    target, draft = _pair()
    B, P, n_new = 4, 96, 40
    ids = torch.randint(3, 32000, (B, P), generator=torch.Generator().manual_seed(3)).cuda()
    plain = target.generate(ids, max_new_tokens=n_new, eos_token_id=[])
    limit = _first_gap_index(target, plain, P)
    for Kp in (1, 4, 7):
        for d in (draft, target):
            got = target.generate(ids, max_new_tokens=n_new, eos_token_id=[], assistant_model=d, num_assistant_tokens=Kp)
            assert torch.equal(got[:, :P], ids)
            for b in range(B):
                diff = torch.nonzero(got[b, P:] != plain[b, P:])
                if len(diff):
                    assert int(diff[0]) >= limit[b], (Kp, b, int(diff[0]), limit[b])
            st = target.engine.assisted_state
            assert (st.graph is not None) == (graph == "1")
            if d is target:
                print("self-draft", Kp, "acceptance", st.acceptance_rate())
                assert st.acceptance_rate() > 0.5
    kw = dict(max_new_tokens=n_new, do_sample=True, top_p=0.9, seed=7, eos_token_id=[], assistant_model=draft, num_assistant_tokens=3)
    assert torch.equal(target.generate(ids, **kw), target.generate(ids, **kw))


def test_draft_without_decode_kernels(monkeypatch):
    """A draft whose head_dim (128) the decode kernels do not take runs its steps on the reference path; the target keeps
    its verify kernels, and the round runs eagerly (no graph)."""
    monkeypatch.setenv("ODB_CUDA_GRAPH", "1")
    target, _ = _pair()
    dcfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=1, num_attention_heads=8, vocab_size=32000)
    assert dcfg.head_dim == 128
    draft = LlamaForCausalLM(dcfg, device="cuda", precision="bf16-mixed", seed=5)
    B, P, n_new = 2, 64, 20
    ids = torch.randint(3, 32000, (B, P), generator=torch.Generator().manual_seed(8)).cuda()
    plain = target.generate(ids, max_new_tokens=n_new, eos_token_id=[])
    limit = _first_gap_index(target, plain, P)
    got = target.generate(ids, max_new_tokens=n_new, eos_token_id=[], assistant_model=draft, num_assistant_tokens=3)
    st = target.engine.assisted_state
    assert st.kernels and not st.graphable and st.graph is None
    for b in range(B):
        diff = torch.nonzero(got[b, P:] != plain[b, P:])
        if len(diff):
            assert int(diff[0]) >= limit[b], (b, int(diff[0]), limit[b])


def test_decode_state_replacement_releases_round_graph(monkeypatch):
    monkeypatch.setenv("ODB_CUDA_GRAPH", "1")
    target, draft = _pair()
    ids = torch.randint(3, 32000, (2, 64), device="cuda")
    target.generate(ids, max_new_tokens=24, eos_token_id=[], assistant_model=draft, num_assistant_tokens=4)
    st = target.engine.assisted_state
    assert st.graph is not None and st.graph_target is target.engine.decode_state
    target.generate(ids, max_new_tokens=200, eos_token_id=[])            # another Smax: a new decode state
    assert st.graph is None and st.graph_target is None


def _our_kernel_names() -> set[str]:
    names = set()
    for src in CSRC.glob("*.cu"):
        names |= set(re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s*)?(\w+)\s*\(", src.read_text()))
    return names


_PROFILE_ROUNDS = r"""
import json, os, sys
import torch
sys.path.insert(0, os.getcwd())
from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.generation import assisted_round
from opendiloco_b200.models.llama import LlamaForCausalLM
tcfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=4, num_attention_heads=16, vocab_size=32000)
target = LlamaForCausalLM(tcfg, device="cuda", precision="bf16-mixed", seed=1)
draft = LlamaForCausalLM(LlamaConfig.from_pretrained("60m"), device="cuda", precision="bf16-mixed", seed=2)
ids = torch.randint(3, 32000, (2, 64), device="cuda")
target.generate(ids, max_new_tokens=24, do_sample=True, top_k=40, eos_token_id=[], assistant_model=draft, num_assistant_tokens=4)
st, tst = target.engine.assisted_state, target.engine.decode_state
from torch.profiler import ProfilerActivity, profile
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(3):
        assisted_round(target, draft, tst, st, 24)
    torch.cuda.synchronize()
print(json.dumps({"graph": st.graph is not None, "cpu": [e.name for e in prof.events()],
                  "gpu": [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]}))
"""


def test_round_is_one_graph_of_our_kernels():
    """Three rounds are three graph launches and no kernel launch, and the GPU runs only our kernels.  The profiler runs
    in a process of its own, so tracing graph replays leaves no profiler state behind for other tests."""
    ours = _our_kernel_names()
    assert {"verify_attn_kernel", "combine_kernel", "accept_kernel", "rope_append_kernel"} <= ours
    env = dict(os.environ, ODB_CUDA_GRAPH="1")
    res = subprocess.run([sys.executable, "-c", _PROFILE_ROUNDS], capture_output=True, text=True, env=env, cwd=ROOT, timeout=600)
    assert res.returncode == 0, res.stderr[-4000:]
    rep = json.loads(res.stdout.strip().splitlines()[-1])
    assert rep["graph"]
    assert sum(n == "cudaGraphLaunch" for n in rep["cpu"]) == 3
    assert not [n for n in rep["cpu"] if n in ("cudaLaunchKernel", "cudaLaunchKernelExC", "cuLaunchKernel", "cuLaunchKernelEx")]
    assert rep["gpu"], "the profiler recorded no GPU activity"
    foreign = [n for n in rep["gpu"] if not any(re.search(rf"\b{k}\b", n) for k in ours)]
    assert not foreign, foreign
    assert any("verify_attn_kernel" in n for n in rep["gpu"]) and any("accept_kernel" in n for n in rep["gpu"])


def test_assisted_generate_does_not_disturb_training_graphs():
    cfg = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4, vocab_size=512)
    dcfg = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=1, num_attention_heads=4, vocab_size=512)
    models = [LlamaForCausalLM(cfg, device="cuda", seed=0), LlamaForCausalLM(dcfg, device="cuda", seed=1)]
    x = torch.randint(3, 512, (4, 128), generator=torch.Generator().manual_seed(0)).cuda()
    for m in models:
        for _ in range(3):
            m.forward_backward(x, x, 1.0)
    key = (4, 128, 1.0, True)
    graphs = [m.engine._graphs[key]["graph"] for m in models]
    ws = [dict(m.engine._ws) for m in models]
    states = [[t.clone() for t in (m.arena.master, m.arena.grad, m.arena.shadow)] for m in models]
    decode_before = models[1].engine.decode_state
    models[0].generate(x[:2, :50], max_new_tokens=30, do_sample=True, seed=1, assistant_model=models[1], num_assistant_tokens=3)
    torch.cuda.synchronize()
    assert models[1].engine.decode_state is decode_before          # the draft's own decode state is not used
    for m, g_obj, w, before in zip(models, graphs, ws, states):
        assert m.engine._graphs[key]["graph"] is g_obj
        assert m.engine._ws == w
        for t0, t1 in zip(before, (m.arena.master, m.arena.grad, m.arena.shadow)):
            assert torch.equal(t0, t1)
    for m, g_obj in zip(models, graphs):
        m.forward_backward(x, x, 1.0)
        assert m.engine._graphs[key]["graph"] is g_obj
