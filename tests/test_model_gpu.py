"""End-to-end model numerics on an H100: the kernel path (CUDA, bf16) against the PyTorch reference path of the same engine."""
import pytest
import torch

from opendiloco_b200 import DiLoCoTrainer, LlamaConfig, LlamaForCausalLM, TrainerConfig

pytestmark = pytest.mark.gpu


def _pair(cfg, seed=0):
    cpu = LlamaForCausalLM(cfg, device="cpu", precision="bf16-mixed", seed=seed)
    gpu = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=seed)
    assert torch.equal(cpu.arena.master, gpu.arena.master.cpu())
    return cpu, gpu


@pytest.mark.parametrize("shape", ["tiny_mha", "wide_gqa"])
def test_forward_backward_matches_reference_path(shape):
    if shape == "tiny_mha":
        cfg = LlamaConfig(hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, vocab_size=1024)
    else:
        cfg = LlamaConfig(hidden_size=512, intermediate_size=1280, num_hidden_layers=2, num_attention_heads=8,
                          num_key_value_heads=2, vocab_size=4096)
    cpu, gpu = _pair(cfg)
    torch.manual_seed(1)
    ids = torch.randint(3, cfg.vocab_size, (2, 128))
    lc = cpu.forward_backward(ids, ids, 1.0)
    lg = gpu.forward_backward(ids.cuda(), ids.cuda(), 1.0)
    assert abs(lc.item() - lg.item()) < 5e-3
    gc, gg = cpu.arena.grad, gpu.arena.grad.cpu()
    assert ((gc - gg).norm() / gc.norm()).item() < 2e-2
    # per-tensor check so one bad kernel cannot hide in the global norm
    worst = max((((cpu.arena.g(n) - gpu.arena.g(n).cpu()).norm() / (cpu.arena.g(n).norm() + 1e-6)).item(), n) for n in cpu.arena.slots)
    print("worst per-tensor rel err vs the bf16 reference path:", worst)
    assert worst[0] < 2e-2, worst


@pytest.mark.parametrize("shape", ["150m_layer", "1b_gqa_layer"])
def test_real_layer_shapes_against_fp32(shape):
    """One decoder layer + embedding + LM head at the Llama-150M / Llama-1B (GQA 32:4) widths and the real vocabulary:
    the bf16 kernel path against the SAME engine run in fp32 (PyTorch ops, fp32 master weights as compute weights)."""
    if shape == "150m_layer":
        cfg = LlamaConfig(hidden_size=1024, intermediate_size=2688, num_hidden_layers=1, num_attention_heads=16, vocab_size=32000)
    else:
        cfg = LlamaConfig(hidden_size=2048, intermediate_size=5632, num_hidden_layers=1, num_attention_heads=32,
                          num_key_value_heads=4, vocab_size=32000)
    ref = LlamaForCausalLM(cfg, device="cuda", precision="32-true", seed=2)
    gpu = LlamaForCausalLM(cfg, device="cuda", precision="bf16-mixed", seed=2)
    assert torch.equal(ref.arena.master, gpu.arena.master)
    torch.manual_seed(3)
    ids = torch.randint(3, cfg.vocab_size, (4, 512), device="cuda")
    lr = ref.forward_backward(ids, ids, 1.0)
    lg = gpu.forward_backward(ids, ids, 1.0)
    assert abs(lr.item() - lg.item()) / lr.item() < 2e-3, (lr.item(), lg.item())
    errs = {n: ((ref.arena.g(n) - gpu.arena.g(n)).norm() / (ref.arena.g(n).norm() + 1e-12)).item() for n in ref.arena.slots}
    worst = max(errs.items(), key=lambda kv: kv[1])
    print(shape, "worst per-tensor rel err vs fp32:", worst, " global:",
          ((ref.arena.grad - gpu.arena.grad).norm() / ref.arena.grad.norm()).item())
    assert worst[1] < 2e-2, errs                       # bf16 activations: a few 1e-3 per tensor is the rounding floor


def test_autograd_facade_on_gpu():
    cfg = LlamaConfig(hidden_size=128, intermediate_size=512, num_hidden_layers=2, num_attention_heads=2, vocab_size=1024)
    a = LlamaForCausalLM(cfg, device="cuda", seed=3)
    b = LlamaForCausalLM(cfg, device="cuda", seed=3)
    ids = torch.randint(3, 1024, (2, 64), device="cuda")
    (a(input_ids=ids, labels=ids).loss / 4).backward()
    b.forward_backward(ids, ids, 0.25)
    assert ((a.arena.grad - b.arena.grad).norm() / b.arena.grad.norm()).item() < 1e-3


def test_training_reduces_loss_and_outer_step_runs():
    cfg = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4, vocab_size=512)
    m = LlamaForCausalLM(cfg, device="cuda", seed=0)
    tr = DiLoCoTrainer(m, TrainerConfig(lr=3e-3, grad_accum=2, local_steps=5, samples_per_step=8, warmup_steps=5, total_steps=200))
    fixed = [{"input_ids": torch.randint(3, 512, (4, 64)).pin_memory()} for _ in range(2)]
    for b in fixed:
        b["labels"] = b["input_ids"]

    def it():
        while True:
            yield from fixed

    g = it()
    losses = [float(tr.train_step(g)) for _ in range(40)]
    assert losses[-1] < losses[0] - 1.0, losses[::8]
    assert tr.optimizer.local_epoch == 8
    sa = tr.optimizer.state_averager
    assert torch.equal(sa.theta_outer, sa.theta_local) is False or tr.real_step % 5 == 0


def test_flagship_shape_step_and_smoke():
    import __graft_entry__ as ge

    ge.smoke()
