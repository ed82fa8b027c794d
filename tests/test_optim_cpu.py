"""FusedAdamW host logic on CPU (reference math path of every kernel): GradScaler on the fused path (K11), clipping
hand-off, hyper-parameter ring.  Reference call sites: train_fsdp.py:390-408, utils.py:124-135."""
import copy

import pytest
import torch

from opendiloco_b200.optim.fused import FusedAdamW
from opendiloco_b200.optim.muon import FusedMuon
from opendiloco_b200.utils.training import found_inf_grad


def _models():
    torch.manual_seed(0)
    a = torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.Linear(32, 8))
    return a, copy.deepcopy(a)


def test_scaled_step_matches_torch_adamw_and_skips_on_overflow():
    ours, ref = _models()
    opt = FusedAdamW(ours.parameters(), lr=1e-2, betas=(0.9, 0.95), weight_decay=0.1, max_grad_norm=1.0)
    ropt = torch.optim.AdamW(ref.parameters(), lr=1e-2, betas=(0.9, 0.95), weight_decay=0.1)
    scaler = torch.amp.GradScaler("cpu", init_scale=1024.0, growth_interval=1000)
    x = torch.randn(4, 16)
    for step in range(3):
        loss = ours(x).pow(2).mean()
        scaler.scale(loss).backward()                       # gradients carry the 1024x loss scale
        rloss = ref(x).pow(2).mean()
        rloss.backward()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), 1.0)
        ropt.step()
        ropt.zero_grad()
        scaled = next(ours.parameters()).grad.clone()
        opt.unscale_(scaler)                                # nothing is rescaled in memory ...
        assert torch.equal(next(ours.parameters()).grad, scaled)
        opt.step_scaled(scaler)                             # ... 1/scale rides into the fused clip + AdamW
        assert not found_inf_grad(opt, scaler)
        scaler.update()
        opt.zero_grad()
        for p, q in zip(ours.parameters(), ref.parameters()):
            assert torch.allclose(p, q, atol=2e-6), (step, (p - q).abs().max())
    # overflow: the update is skipped, the scaler backs off
    before = [p.detach().clone() for p in ours.parameters()]
    loss = ours(x).pow(2).mean()
    scaler.scale(loss).backward()
    next(ours.parameters()).grad[0, 0] = float("inf")
    opt.unscale_(scaler)
    opt.step_scaled(scaler)
    assert found_inf_grad(opt, scaler)
    scale_before = scaler.get_scale()
    scaler.update()
    assert scaler.get_scale() == scale_before * 0.5
    for p, q in zip(ours.parameters(), before):
        assert torch.equal(p, q)


def test_hp_ring_slots_are_not_reused_while_in_flight():
    ours, _ = _models()
    opt = FusedAdamW(ours.parameters(), lr=1e-3)
    seen = set()
    for i in range(2 * opt.HP_RING):
        for p in ours.parameters():
            p.grad = torch.ones_like(p)
        opt.param_groups[0]["lr"] = 1e-3 * (i + 1)
        slot = opt._hp_slot
        opt.step()
        seen.add(slot)
        assert abs(float(opt._hp[0]) - 1e-3 * (i + 1)) < 1e-9
    assert seen == set(range(opt.HP_RING))


# ------------------------------------------------------------------------------------------------ skipped steps
# A GradScaler overflow step is not an AdamW step: torch's GradScaler.step does not call optimizer.step(), so
# state["step"] and the bias corrections 1 - beta^t only count the updates applied.  FusedAdamW (and FusedMuon's AdamW
# part) must follow, including across save / load.  The reference is torch.optim.AdamW + GradScaler in float64, fed the
# same gradients; ours runs in fp32, so it may differ by fp32 rounding (TRAJ_TOL: < 1e-6 measured over these 10 steps),
# while counting the skipped step moves every later update by ~25 % of lr (2.6e-3 here).
TRAJ_TOL = 1e-5
DEVICES = ["cpu", pytest.param("cuda", marks=pytest.mark.gpu)]


def _scaler_run(device: str, muon: bool, overflow_steps: tuple[int, ...], n_steps: int = 10, save_at: int = 5):
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(16, 32), torch.nn.Linear(32, 8)).to(device)
    ref = copy.deepcopy(model).double()
    kw = dict(lr=1e-2, weight_decay=0.1)

    def make(m):
        if muon:     # weight matrices take Muon, biases AdamW
            return FusedMuon(m.parameters(), adamw_betas=(0.9, 0.95), **kw)
        return FusedAdamW(m.parameters(), betas=(0.9, 0.95), **kw)

    opt = make(model)
    compared = [i for i, p in enumerate(ref.parameters()) if not muon or p.ndim == 1]
    rparams = [p for i, p in enumerate(ref.parameters()) if i in compared]
    ropt = torch.optim.AdamW(rparams, betas=(0.9, 0.95), **kw)
    scaler = torch.amp.GradScaler(device, init_scale=1024.0, growth_interval=1000)
    rscaler = torch.amp.GradScaler(device, init_scale=1024.0, growth_interval=1000)
    rscaler.scale(torch.ones((), dtype=torch.float64, device=device))     # initialises the scale on the device
    gen = torch.Generator().manual_seed(1)
    for step in range(n_steps):
        if step == save_at:        # checkpoint round trip into a fresh model + optimizer, then carry on
            sd = opt.state_dict()
            model = copy.deepcopy(model)
            opt = make(model)
            opt.load_state_dict(sd)
        scale = scaler.get_scale()
        assert scale == rscaler.get_scale()
        ours = list(model.parameters())
        for p, rp in zip(ours, ref.parameters()):
            g = torch.randn(p.shape, generator=gen, dtype=torch.float64) * 0.1
            if step in overflow_steps and p is ours[-1]:
                g.view(-1)[-1] = float("inf")            # the last element of the last parameter only
            p.grad.copy_((g * scale).float().to(device))
            rp.grad = (g * scale).to(device)
        before = [p.detach().clone() for p in ours]
        opt.unscale_(scaler)
        opt.step_scaled(scaler)
        scaler.update()
        rscaler.step(ropt)
        rscaler.update()
        opt.zero_grad()
        ropt.zero_grad()
        if step in overflow_steps:
            assert all(torch.equal(p, b) for p, b in zip(ours, before)), step
        for i in compared:
            err = (ours[i].double() - list(ref.parameters())[i]).abs().max().item()
            assert err <= TRAJ_TOL, (step, i, err)
    applied = n_steps - len(overflow_steps)
    assert opt.applied_steps() == applied
    sd = opt.state_dict()
    steps = [float(st["step"]) for st in sd["state"].values() if "step" in st]
    assert steps and all(s == applied for s in steps), steps
    assert all(float(ropt.state[p]["step"]) == applied for p in rparams)


@pytest.mark.parametrize("device", DEVICES)
@pytest.mark.parametrize("muon", [False, True], ids=["adamw", "muon"])
@pytest.mark.parametrize("overflow_steps", [(0,), (3,), (0, 7)], ids=["first", "mid", "first+after_load"])
def test_overflow_step_is_not_counted_as_an_adamw_step(device, muon, overflow_steps):
    _scaler_run(device, muon, overflow_steps)
