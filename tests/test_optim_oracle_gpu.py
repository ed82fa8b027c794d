"""Element-by-element oracle for the sm_90a optimizer, outer-step and 8-bit codec kernels (csrc/optim.cu, the AdamW part of
csrc/muon.cu, csrc/quant.cu), each against a float64 or exact reference written here and fed the exact fp32 / bf16
values the kernel reads.

Every check is a one-step oracle: the reference starts from the kernel's own state (p, m, v or theta_outer, buf) copied
to float64, advances one step, and only that step is compared.  Bounds are derived, not fitted: each is a count of
fp32 unit roundoffs U = 2^-24 times the magnitude of the terms the kernel rounds (``scale``), so an element whose terms
cancel is not held to a relative bound it cannot meet, and an exactly-zero result must be exactly zero.  Where no
rounding choice exists (copies, comparisons, one correctly rounded operation, round-to-nearest-even casts, integer sums)
the check is bit for bit.

Measured on an H100 80GB HBM3 (700 W power limit), CUDA 12.9, torch 2.11: the worst ratio err / (U x scale + 2^-149) of
every bound is given beside it.  The five DiLoCo rounds stay below 2.3e-8 against a limit of 9.5e-7.
"""
import math

import numpy as np
import pytest
import torch

from opendiloco_b200.ops import kernels as K
from opendiloco_b200.ops import muon as M
from opendiloco_b200.parallel import compression as C

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
U = 2.0 ** -24
# a rounding whose result falls in fp32's subnormal range errs by up to half of 2^-149 absolutely, not U relatively (a
# clipped 1e-12 gradient squared into v is ~1e-41): every bound gets that absolute allowance per counted rounding
TINY = 2.0 ** -149

# fp32 sum of squares of the gradient (grad_sqnorm: per-thread chains, warp and block trees, then adamw_step's re-reduction
# of <= 2048 partials): its relative error is at most (longest chain of additions) x U, < 40 U for every n below.
# The norm, the clip coefficient and therefore every clipped gradient inherit it.           measured: norm 0.52, clip 1.07
NORM_C = 64
BOUND = {
    # m' = m + (1 - b1)(g' - m): 3 roundings of terms <= b1|m| + (1 - b1)|g'|, plus the clip coefficient's NORM_C
    "m": 4 + NORM_C,                                                                      # measured 1.84
    # v' = b2 v + (1 - b2) g'^2: 4 roundings of positive terms, g'^2 doubles the clip coefficient's error
    "v": 6 + 2 * NORM_C,                                                                  # measured 3.67
    # p' = p (1 - lr wd) - (lr / bc1) m' / (sqrt(v') / sqrt(bc2) + eps): m' as above, ~9 U through the denominator and
    # division, 3 U on the decay and the final subtraction; scale = |p (1 - lr wd)| + (lr / bc1) (b1|m| + (1 - b1)|g'|) / denom
    "p": 16 + NORM_C,                                                                     # measured 2.99
    # buf' = mu buf + d (d = delta * dscale, fused form: one more rounding for theta_outer - theta_local)
    "buf": 4,                                                                             # measured 1.79
    # theta' = theta - lr (d + mu buf') (nesterov) or theta - lr buf': scale = |theta| + lr (|d| + mu (mu|buf| + |d|))
    "theta": 8,                                                                           # measured 2.56
}


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _check(name, got, ref, scale, c):
    """|got - ref| <= c (U scale + 2^-149) for every element (got: kernel output, ref / scale: float64)."""
    got = got.detach().double()
    err = (got - ref).abs()
    lim = c * (U * scale + TINY)
    ratio = float((err / (U * scale + TINY)).max())
    print(f"[bound] {name}: worst {ratio:.2f} U (limit {c})")
    bad = ~(err <= lim)
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError(f"{name}: {int(bad.sum())} of {err.numel()} elements over {c} (U x scale + 2^-149); first at {i}: "
                             f"got {float(got[i])!r} ref {float(ref[i])!r} scale {float(scale[i])!r}")


# ------------------------------------------------------------------------------------------------ AdamW
def _hp(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, wd=0.1, t=1, max_norm=0.0, inv_scale=1.0) -> torch.Tensor:
    hp = torch.zeros(K.HP_SIZE, dtype=torch.float32)
    for k, v in K.adamw_hp(lr, betas, eps, wd, t, max_norm).items():
        hp[k] = v
    hp[K.HP_INVSCALE] = inv_scale
    return hp.to(DEV)


def _mixed_grad(n, seed, scale=1.0):
    """N(0, 1) times magnitudes spread over 10^-12 .. 10^4, with exact zeros: mixed magnitudes in one arena."""
    g = _gen(seed)
    mag = 10.0 ** (torch.rand(n, device=DEV, generator=g) * 16 - 12)
    x = torch.randn(n, device=DEV, generator=g) * mag
    x[::97] = 0.0
    x[1::101] = 1e-12
    x[2::103] = -1e4
    return (x * scale).contiguous()


def _state(n, g, seed, t):
    """(p, m, v): zero moments at step 1, moments of the gradient's size later."""
    gen = _gen(seed + 1)
    p = torch.randn(n, device=DEV, generator=gen)
    if t == 1:
        return p, torch.zeros_like(p), torch.zeros_like(p)
    m = g * torch.randn(n, device=DEV, generator=gen) * 0.3
    v = (g * g) * torch.rand(n, device=DEV, generator=gen) * 2
    return p, m, v


def _adamw_ref(p, g, m, v, hp, bc=None):
    """One fp64 AdamW step (torch semantics) from the kernel's inputs; returns p', m', v' and their error scales."""
    lr, b1, b2, eps, wd, bc1, bc2, max_norm, inv_scale = (float(x) for x in hp[:9].cpu())
    if bc is not None:
        bc1, bc2 = bc
    p, g, m, v = (t.double() for t in (p, g, m, v))
    gnorm = float(g.norm()) * inv_scale
    clip = min(1.0, max_norm / (gnorm + 1e-6)) if max_norm > 0 else 1.0
    gr = g * (inv_scale * clip)
    m1 = m + (1 - b1) * (gr - m)
    v1 = b2 * v + (1 - b2) * gr * gr
    denom = v1.sqrt() / math.sqrt(bc2) + eps
    pd = p * (1 - lr * wd)
    p1 = pd - (lr / bc1) * m1 / denom
    m_scale = b1 * m.abs() + (1 - b1) * gr.abs()
    v_scale = b2 * v + (1 - b2) * gr * gr
    p_scale = pd.abs() + (lr / bc1) * m_scale / denom
    return (p1, m1, v1), (p_scale, m_scale, v_scale), (gnorm, clip)


def _run_adamw(p, g, m, v, hp, shadow, zero_grad, found_inf=None, skipped=None):
    partials = torch.zeros(K.MAX_PARTIALS, device=DEV)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    npart = K.grad_sqnorm(g, partials, flag)
    stats = torch.zeros(2, device=DEV)
    K.adamw_step(p, g, m, v, shadow, hp, partials, npart, found_inf, stats, zero_grad=zero_grad, skipped=skipped)
    torch.cuda.synchronize()
    return stats, flag


ADAMW_CASES = {
    # name: (n, t, lr, max_norm, inv_scale)
    "step1_clipped_scaled": (1 << 16, 1, 1e-3, 1.0, 2.0 ** -16),
    "step1e4_unclipped": (1 << 16, 10_000, 1e-3, 1e30, 1.0),
    "lr0": (4096, 5, 0.0, 1.0, 1.0),
    "n4": (4, 3, 1e-2, 0.0, 1.0),
    "strided": ((1 << 22) + 12, 2, 1e-3, 1.0, 2.0 ** -16),   # > 4 float4 strides per thread of the 1056-CTA grid
}
VARIANTS = [(True, True), (True, False), (False, True), (False, False)]


@pytest.mark.parametrize("shadow_on,zero_grad", VARIANTS, ids=["shadow-zero", "shadow", "zero", "plain"])
@pytest.mark.parametrize("case", list(ADAMW_CASES))
def test_adamw_step_against_fp64(case, shadow_on, zero_grad):
    n, t, lr, max_norm, inv_scale = ADAMW_CASES[case]
    g = _mixed_grad(n, 10 + n % 7, scale=1.0 / inv_scale)
    p, m, v = _state(n, g * inv_scale, 20, t)
    hp = _hp(lr=lr, t=t, max_norm=max_norm, inv_scale=inv_scale)
    (p1, m1, v1), (ps, ms, vs), (gnorm, clip) = _adamw_ref(p, g, m, v, hp)
    g0, p0 = g.clone(), p.clone()
    shadow = torch.full((n,), 7.0, dtype=BF, device=DEV) if shadow_on else None
    stats, flag = _run_adamw(p, g, m, v, hp, shadow, zero_grad)
    assert int(flag) == 0
    if max_norm > 0:
        assert clip < 1.0 or max_norm > 1e20, "the clipped cases must actually clip"
    _check(f"{case}/norm", stats[0:1], torch.tensor([gnorm], dtype=torch.float64, device=DEV),
           torch.tensor([gnorm], dtype=torch.float64, device=DEV), NORM_C)
    _check(f"{case}/clip", stats[1:2], torch.tensor([clip], dtype=torch.float64, device=DEV),
           torch.tensor([clip], dtype=torch.float64, device=DEV), NORM_C + 4)
    _check(f"{case}/m", m, m1, ms, BOUND["m"])
    _check(f"{case}/v", v, v1, vs, BOUND["v"])
    if lr == 0.0:
        assert torch.equal(p, p0), "lr = 0 must leave the weights bit-identical"
    _check(f"{case}/p", p, p1, ps, BOUND["p"])
    if shadow_on:
        assert torch.equal(shadow, p.to(BF))
    assert torch.equal(g, torch.zeros_like(g)) if zero_grad else torch.equal(g, g0)


@pytest.mark.parametrize("shadow_on,zero_grad", VARIANTS, ids=["shadow-zero", "shadow", "zero", "plain"])
def test_adamw_step_skips_on_a_non_finite_last_element(shadow_on, zero_grad):
    """grad_sqnorm flags a non-finite value in the very last element; the step then leaves p, m, v (and the shadow)
    bit-identical, still zeroes the gradient, and counts the skip in the device counter."""
    n = (1 << 20) + 8
    g = _mixed_grad(n, 3)
    p, m, v = _state(n, g, 4, 7)
    for bad in (float("inf"), float("nan")):
        g[-1] = bad
        shadow = torch.full((n,), 7.0, dtype=BF, device=DEV) if shadow_on else None
        before = [t.clone() for t in (p, m, v, g)]
        sh0 = None if shadow is None else shadow.clone()
        skipped = torch.tensor([0, 3], dtype=torch.int32, device=DEV)     # step 7 reads slot 1, writes slot 0
        partials = torch.zeros(K.MAX_PARTIALS, device=DEV)
        flag = torch.zeros(1, dtype=torch.int32, device=DEV)
        npart = K.grad_sqnorm(g, partials, flag)
        K.adamw_step(p, g, m, v, shadow, _hp(t=7, max_norm=1.0), partials, npart, flag, None, zero_grad=zero_grad,
                     skipped=skipped)
        torch.cuda.synchronize()
        assert int(flag) == 1, bad
        for a, b in zip((p, m, v), before):
            assert torch.equal(a, b)
        if shadow_on:
            assert torch.equal(shadow, sh0)
        if zero_grad:
            assert torch.equal(g, torch.zeros_like(g))
        else:
            assert torch.equal(g[:-1], before[3][:-1])
            g.copy_(before[3])
        assert skipped.tolist() == [4, 3]


@pytest.mark.parametrize("found", [0, 1])
def test_adamw_bias_correction_counts_only_applied_updates(found):
    """After s skipped steps, host step t is update t - s: the kernels recompute 1 - beta^(t - s) in double."""
    n, t, s = 8192, 10, 4
    g = _mixed_grad(n, 5)
    p, m, v = _state(n, g, 6, 2)
    hp = _hp(lr=1e-2, betas=(0.9, 0.999), t=t)
    b1, b2 = 0.9, 0.999
    (p1, m1, v1), (ps, ms, vs), _ = _adamw_ref(p, g, m, v, hp, bc=(1 - b1 ** (t - s), 1 - b2 ** (t - s)))
    skipped = torch.tensor([s, 99], dtype=torch.int32, device=DEV)          # t even: slot 0 is read, slot 1 written
    fi = torch.tensor([found], dtype=torch.int32, device=DEV)
    p0 = p.clone()
    K.adamw_step(p, g.clone(), m, v, None, hp, torch.zeros(K.MAX_PARTIALS, device=DEV), 0, fi, None, zero_grad=True,
                 skipped=skipped)
    torch.cuda.synchronize()
    assert skipped.tolist() == [s, s + found]
    if found:
        assert torch.equal(p, p0)
    else:
        _check("bias_corr/m", m, m1, ms, BOUND["m"])
        _check("bias_corr/p", p, p1, ps, BOUND["p"])


# ------------------------------------------------------------------------------------------------ adamw_segments
# aligned (float4) and unaligned (scalar) chunks of one arena, in one launch
SEGMENTS = [(0, 1024), (1027, 1), (1030, 509), (2048, 1021), (3072, 4096), (7171, 6), (8192, 4092)]


@pytest.mark.parametrize("shadow_on,zero_grad", [(True, True), (False, False)], ids=["shadow-zero", "plain"])
def test_adamw_segments_against_fp64_and_adamw_step(shadow_on, zero_grad):
    n = 12288
    g = _mixed_grad(n, 7, scale=2.0 ** 16)
    p, m, v = _state(n, g * 2.0 ** -16, 8, 3)
    hp = _hp(lr=1e-3, wd=0.1, t=3, max_norm=1.0, inv_scale=2.0 ** -16)
    (p1, m1, v1), (ps, ms, vs), _ = _adamw_ref(p, g, m, v, hp)
    covered = torch.zeros(n, dtype=torch.bool, device=DEV)
    for o, ln in SEGMENTS:
        covered[o:o + ln] = True
    # the same step by adamw_step on a copy (every element)
    q, gq, mq, vq = p.clone(), g.clone(), m.clone(), v.clone()
    _run_adamw(q, gq, mq, vq, hp, None, False)
    before = [t.clone() for t in (p, g, m, v)]
    shadow = torch.full((n,), 7.0, dtype=BF, device=DEV) if shadow_on else None
    partials = torch.zeros(K.MAX_PARTIALS, device=DEV)
    flag = torch.zeros(1, dtype=torch.int32, device=DEV)
    npart = K.grad_sqnorm(g, partials, flag)
    chunks = torch.tensor(SEGMENTS, dtype=torch.int64, device=DEV)
    M.adamw_segments(p, g, m, v, shadow, chunks, hp, partials, npart, None, zero_grad)
    torch.cuda.synchronize()
    c = covered
    _check("segments/m", m[c], m1[c], ms[c], BOUND["m"])
    _check("segments/v", v[c], v1[c], vs[c], BOUND["v"])
    _check("segments/p", p[c], p1[c], ps[c], BOUND["p"])
    _check("segments_vs_step/p", p[c], q[c].double(), ps[c], 2 * BOUND["p"])
    for a, b in zip((p, g, m, v), before):             # outside the chunks nothing moves
        assert torch.equal(a[~c], b[~c])
    if shadow_on:
        assert torch.equal(shadow[c], p[c].to(BF)) and bool((shadow[~c] == 7.0).all())
    assert torch.equal(g[c], torch.zeros_like(g[c])) if zero_grad else torch.equal(g, before[1])


@pytest.mark.parametrize("found", [0, 1])
def test_adamw_segments_skip_and_bias_correction(found):
    n = 12288
    g = _mixed_grad(n, 9)
    p, m, v = _state(n, g, 10, 2)
    t, s = 9, 2
    hp = _hp(lr=1e-2, t=t)
    (p1, _, _), (ps, _, _), _ = _adamw_ref(p, g, m, v, hp, bc=(1 - 0.9 ** (t - s), 1 - 0.999 ** (t - s)))
    skipped = torch.tensor([0, s], dtype=torch.int32, device=DEV)            # t odd: slot 1 is read, slot 0 written
    fi = torch.tensor([found], dtype=torch.int32, device=DEV)
    before = [x.clone() for x in (p, m, v)]
    chunks = torch.tensor(SEGMENTS, dtype=torch.int64, device=DEV)
    M.adamw_segments(p, g, m, v, None, chunks, hp, torch.zeros(K.MAX_PARTIALS, device=DEV), 0, fi, True, skipped=skipped)
    torch.cuda.synchronize()
    assert skipped.tolist() == [s + found, s]
    c = torch.zeros(n, dtype=torch.bool, device=DEV)
    for o, ln in SEGMENTS:
        c[o:o + ln] = True
    if found:
        for a, b in zip((p, m, v), before):
            assert torch.equal(a, b)
    else:
        _check("segments_bias_corr/p", p[c], p1[c], ps[c], BOUND["p"])
    assert bool((g[c] == 0).all())


# ------------------------------------------------------------------------------------------------ outer step
def _edge_floats(n, seed):
    """N(0, 1) with subnormals, exact cancellations (a == b) and infinities mixed in."""
    g = _gen(seed)
    a = torch.randn(n, device=DEV, generator=g)
    b = a + torch.randn(n, device=DEV, generator=g) * 1e-3
    b[::5] = a[::5]                                     # a - b == 0 exactly
    a[1::7] = 3e-39                                     # subnormal operands and results
    b[1::7] = 1e-39
    a[2::11] = float("inf")
    b[3::13] = float("-inf")
    b[4::17] = -a[4::17]
    return a, b


def test_pseudo_grad_fp32_and_bf16_bit_exact():
    n = (1 << 20) + 4
    a, b = _edge_floats(n, 1)
    ref = a.cpu() - b.cpu()                             # one correctly rounded subtraction (subnormals kept)
    d32 = torch.empty(n, device=DEV)
    d16 = torch.empty(n, dtype=BF, device=DEV)
    K.pseudo_grad(a, b, d32)
    K.pseudo_grad(a, b, d16)
    assert torch.equal(d32.cpu().view(torch.int32), ref.view(torch.int32))
    r16 = ref.to(BF)
    nan = torch.isnan(r16)
    assert torch.equal(torch.isnan(d16.cpu()), nan)
    assert torch.equal(d16.cpu()[~nan].view(torch.int16), r16[~nan].view(torch.int16))


def _nesterov_ref(to, buf, d, lr, mu, nesterov):
    to, buf, d = to.double(), buf.double(), d.double()
    b1 = mu * buf + d
    step = d + mu * b1 if nesterov else b1
    t1 = to - lr * step
    buf_scale = mu * buf.abs() + d.abs()
    t_scale = to.abs() + lr * (d.abs() + mu * buf_scale) if nesterov else to.abs() + lr * buf_scale
    return (t1, b1), (t_scale, buf_scale)


@pytest.mark.parametrize("nesterov", [True, False], ids=["nesterov", "momentum"])
@pytest.mark.parametrize("form", ["fused", "fp32", "bf16"])
def test_nesterov_outer_against_fp64(form, nesterov):
    n = (1 << 18) + 4
    g = _gen(2)
    to = torch.randn(n, device=DEV, generator=g)
    tl = to - torch.randn(n, device=DEV, generator=g) * 1e-2
    buf = torch.randn(n, device=DEV, generator=g) * 1e-2
    lr, mu, dscale = 0.7, 0.9, 1.0 / 3.0
    ds = float(torch.tensor(dscale, dtype=torch.float32))           # the fp32 value the kernel multiplies by
    if form == "fused":
        delta = None
        d = (to.double() - tl.double()) * ds
    else:
        delta = (torch.randn(n, device=DEV, generator=g) * 1e-2).to(torch.float32 if form == "fp32" else BF)
        d = delta.double() * ds
    (t1, b1), (ts, bs) = _nesterov_ref(to, buf, d, float(torch.tensor(lr, dtype=torch.float32)),
                                       float(torch.tensor(mu, dtype=torch.float32)), nesterov)
    shadow = torch.empty(n, dtype=BF, device=DEV)
    K.nesterov_outer(to, buf, delta, tl, shadow, lr, mu, nesterov, dscale)
    torch.cuda.synchronize()
    _check(f"nesterov_{form}/buf", buf, b1, bs, BOUND["buf"])
    _check(f"nesterov_{form}/theta", to, t1, ts, BOUND["theta"])
    assert torch.equal(tl, to)
    assert torch.equal(shadow, to.to(BF))


def test_diloco_outer_rounds_against_fp64_loop():
    """Five outer rounds of DiLoCoOptimizer on one GPU (fused single-worker Nesterov step) against an fp64 outer loop fed
    the theta_local each round ended with.  The reference keeps its own fp64 theta_outer, so the fp32 roundings of
    earlier rounds add up: at most ROUNDS x BOUND["theta"] U of the largest |theta|."""
    from functools import partial

    from opendiloco_b200.optim.fused import FusedAdamW
    from opendiloco_b200.parallel.diloco import DiLoCoOptimizer

    class Recording(FusedAdamW):
        def step(self, *a, **k):
            out = super().step(*a, **k)
            self.theta_local = self.fv.flat.detach().double().clone()      # what the outer step of this call will read
            return out

    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.Tanh(), torch.nn.Linear(128, 8)).to(DEV)
    H, rounds, lr, mu = 3, 5, 0.7, 0.9
    opt = DiLoCoOptimizer(batch_size=32, num_inner_steps=H, params=model.parameters(),
                          outer_optimizer=partial(torch.optim.SGD, lr=lr, momentum=mu, nesterov=True),
                          inner_optimizer=partial(Recording, lr=1e-2, weight_decay=0.1, betas=(0.9, 0.95)))
    inner = opt.inner_optimizer
    theta = inner.fv.flat.detach().double().clone()
    buf = torch.zeros_like(theta)
    lr32, mu32 = float(torch.tensor(lr, dtype=torch.float32)), float(torch.tensor(mu, dtype=torch.float32))
    for r in range(rounds):
        for _ in range(H):
            x, y = torch.randn(32, 64, device=DEV), torch.randn(32, 8, device=DEV)
            torch.nn.functional.mse_loss(model(x), y).backward()
            opt.step()
            opt.zero_grad()
        d = theta - inner.theta_local
        buf = mu32 * buf + d
        theta = theta - lr32 * (d + mu32 * buf)
        got = opt.state_averager.theta_outer.double()
        err = float((got - theta).abs().max())
        lim = (r + 1) * BOUND["theta"] * U * float(theta.abs().max())
        print(f"[bound] diloco round {r}: err {err:.3e} limit {lim:.3e}")
        assert err <= lim, (r, err, lim)
        assert torch.equal(inner.fv.flat, opt.state_averager.theta_outer)
    assert opt.local_epoch == rounds


# ------------------------------------------------------------------------------------------------ checksum
@pytest.mark.parametrize("n", [1 << 24, (1 << 20) + 3], ids=["large", "fallback_n_mod_4"])
def test_checksum_i32_exact(n):
    g = torch.Generator().manual_seed(3)
    words = torch.randint(-(2 ** 31), 2 ** 31 - 1, (n,), dtype=torch.int32, generator=g)
    words[:64] = -(2 ** 31)                              # sign bit set, the most negative word
    expect = int(words.numpy().astype(np.int64).sum())   # |sum| < 2^55: no wrap in int64
    got = K.checksum_i32(words.to(DEV).view(torch.float32))
    assert int(got.item()) == expect


# ------------------------------------------------------------------------------------------------ 8-bit codecs
def _cpu_blockwise(x):
    return C.BlockwiseQuantization().compress(x.cpu())


def test_blockwise8_codes_identical_to_cpu_and_dequant_bound():
    nb = 64
    g = _gen(4)
    x = torch.randn(nb, C.QBLOCK, device=DEV, generator=g) * (10.0 ** torch.linspace(-6, 4, nb, device=DEV))[:, None]
    x[3] = 0.0                                            # an all-zero block
    x[5::7, 17] = 1e6                                     # one outlier per block
    x[9] = 0.25 * torch.randint(-4, 5, (C.QBLOCK,), device=DEV, generator=g)
    x[9, 0] = 127.0                                       # absmax 127: scale 1, so x = k + 0.5 are exact half steps
    x[9, 1:8] = torch.tensor([0.5, 1.5, 2.5, -0.5, -1.5, 3.5, -3.5], device=DEV)
    x = x.reshape(-1).contiguous()
    codec = C.BlockwiseQuantization()
    q, absmax = codec.compress(x)
    qc, ac = _cpu_blockwise(x)
    assert torch.equal(absmax.cpu(), ac)
    assert torch.equal(q.cpu(), qc)
    assert q[3 * C.QBLOCK:4 * C.QBLOCK].eq(0).all() and float(absmax[3]) == 0.0
    assert q[9 * C.QBLOCK + 1:9 * C.QBLOCK + 8].tolist() == [0, 2, 2, 0, -2, 4, -4]        # ties to even
    out = torch.empty_like(x)
    codec.decompress_into(q, absmax, out)
    am = absmax.double().repeat_interleave(C.QBLOCK)
    # half a code step, plus the rounding of x * (127 / absmax) (2 U of a code step of 127) and of q * (absmax / 127)
    # (2 U of |deq| <= absmax)
    err = (out.double() - x.double()).abs()
    lim = am / 254 + 4 * U * am
    assert bool((err <= lim).all()), float((err - lim).max())
    assert bool((out[3 * C.QBLOCK:4 * C.QBLOCK] == 0).all())
    # accumulate with alpha: out0 + alpha * q * absmax / 127, against fp64 of the exact codes
    base = torch.randn(x.numel(), device=DEV, generator=g)
    out = base.clone()
    alpha = 1.0 / 3.0
    codec.decompress_into(q, absmax, out, alpha=alpha, accumulate=True)
    val = q.double() * am * alpha / 127
    _check("blockwise8/accumulate", out, base.double() + val, base.double().abs() + val.abs(), 4)


def test_affine8_codes_match_cpu_path():
    n = (1 << 20) + 5
    g = _gen(5)
    x = torch.randn(n, device=DEV, generator=g) * 0.02 + 0.001
    x[::1000] = 10.0                                      # hundreds of buckets beyond +128: clamp to 255
    x[1::1000] = -10.0                                    # ... and to 0
    mean = x.mean()
    scale = 6 * (x - mean).pow(2).mean().sqrt() / 256
    ms = torch.stack([mean, scale]).float()
    q = torch.empty(n, dtype=torch.uint8, device=DEV)
    C._call("odb_quant_affine8", x.data_ptr(), q.data_ptr(), n, ms.data_ptr(), torch.cuda.current_stream().cuda_stream)
    xc, mc, sc = x.cpu(), ms[0].cpu(), float(ms[1])
    ref = (torch.round((xc - mc) * (1.0 / sc)) + 128).clamp(0, 255).to(torch.uint8)      # the codec's CPU path
    diff = (q.cpu().int() - ref.int()).abs()
    # the CPU path rounds 1 / scale from double, the kernel divides in fp32: codes may differ by one only where the
    # value lies within an fp32 ulp or so of a .5 boundary
    z = (xc.double() - float(mc)) / sc
    near_half = ((z - z.floor() - 0.5).abs() <= 4 * U * z.abs().clamp_min(1.0))
    assert int(diff.max()) <= 1 and bool(near_half[diff == 1].all()), int((diff == 1).sum())
    assert bool((q[::1000] == 255).all()) and bool((q[1::1000] == 0).all())
    # std = 0: every code is 128
    ms0 = torch.tensor([0.5, 0.0], device=DEV)
    c0 = torch.zeros(4096, dtype=torch.uint8, device=DEV)
    C._call("odb_quant_affine8", torch.full((4096,), 0.5, device=DEV).data_ptr(), c0.data_ptr(), 4096, ms0.data_ptr(),
            torch.cuda.current_stream().cuda_stream)
    assert bool((c0 == 128).all())


def _bucket8(x, borders):
    q = torch.empty(x.numel(), dtype=torch.uint8, device=DEV)
    C._call("odb_quant_bucket8", x.data_ptr(), q.data_ptr(), x.numel(), borders.data_ptr(),
            torch.cuda.current_stream().cuda_stream)
    return q


def test_bucket8_identical_to_torch_bucketize():
    n = (1 << 20) + 7
    g = _gen(6)
    x = torch.randn(n, device=DEV, generator=g)
    x[::3] = 0.0                                          # a pseudo-gradient with many exact zeros
    x[1::29] = -0.0
    srt = x[::4].sort().values
    borders = srt[(torch.linspace(0, 1, 257, device=DEV)[1:-1] * (srt.numel() - 1)).round().long()].contiguous()
    assert int((borders == 0).sum()) > 50                 # a long run of duplicate borders
    x[2::31] = borders[torch.randint(0, 255, (x[2::31].numel(),), device=DEV, generator=g)]     # x equal to a border
    x[5] = float("inf")
    x[6] = float("-inf")
    x[7] = borders[0]
    x[8] = borders[-1]
    q = _bucket8(x, borders)
    ref = torch.bucketize(x.cpu(), borders.cpu(), right=True)
    assert torch.equal(q.cpu().long(), ref)
    # strictly increasing borders too: every one of the 256 codes is reachable
    b2 = torch.linspace(-3, 3, 255, device=DEV)
    y = torch.cat([b2, b2 - 1e-3, torch.randn(1 << 16, device=DEV, generator=g) * 2]).contiguous()
    assert torch.equal(_bucket8(y, b2).cpu().long(), torch.bucketize(y.cpu(), b2.cpu(), right=True))


def test_bucket_stats_and_lookup_against_fp64():
    """Counts are exact integers (one bucket holds more than 2^24 members); sums are fp32 atomics in an arbitrary order,
    bounded by (the longest chain of additions) x U x the bucket's sum of |x|; every decoded value lies in its bucket's
    [min, max] up to that bound."""
    n = (1 << 24) + (1 << 22)
    g = _gen(7)
    x = torch.zeros(n, device=DEV)
    nz = torch.rand(n, device=DEV, generator=g) < 0.05
    x[nz] = torch.randn(int(nz.sum()), device=DEV, generator=g) * 1e-3
    codec = C.Quantile8BitQuantization()
    q, table = codec.compress(x)
    qc = q.long().cpu()
    xc = x.double().cpu()
    cnt = torch.bincount(qc, minlength=256)
    assert int(cnt.max()) > (1 << 24)
    sums = torch.zeros(256, dtype=torch.float64).index_add_(0, qc, xc)
    abs_sums = torch.zeros(256, dtype=torch.float64).index_add_(0, qc, xc.abs())
    # the codec only keeps sums / counts, and the big bucket's sum is 0: check the statistics kernel's outputs directly
    s_k = torch.zeros(256, device=DEV)
    c_k = torch.zeros(256, dtype=torch.int32, device=DEV)
    C._call("odb_bucket_stats", x.data_ptr(), q.data_ptr(), n, s_k.data_ptr(), c_k.data_ptr(), torch.cuda.current_stream().cuda_stream)
    assert torch.equal(c_k.cpu().long(), cnt)
    grid = min(-(-n // 2048), 132 * 8)
    chain = (cnt + grid).double()                          # per-CTA chain + one global add per CTA
    _check("bucket_stats/sum", s_k.cpu(), sums, chain * abs_sums, 1.0)
    lo = torch.full((256,), math.inf, dtype=torch.float64).scatter_reduce_(0, qc, xc, "amin")
    hi = torch.full((256,), -math.inf, dtype=torch.float64).scatter_reduce_(0, qc, xc, "amax")
    used = cnt > 0
    slack = (chain * U * abs_sums / cnt.clamp_min(1) + 2 * U * torch.maximum(lo.abs(), hi.abs()))[used]
    t = table.double().cpu()[used]
    assert bool(((t >= lo[used] - slack) & (t <= hi[used] + slack)).all())
    # lookup: out = table[q] * alpha, optionally accumulated
    out = torch.empty_like(x)
    codec.decompress_into(q, table, out)
    assert torch.equal(out.cpu(), table.cpu()[qc])
    base = torch.randn(n, device=DEV, generator=g)
    out = base.clone()
    codec.decompress_into(q, table, out, alpha=0.25, accumulate=True)
    val = table.double().cpu()[qc] * 0.25
    _check("lookup8/accumulate", out.cpu(), base.double().cpu() + val, base.double().cpu().abs() + val.abs(), 2)


@pytest.mark.parametrize("name", ["none", "fp16", "bf16", "scaled-fp16", "uniform8bit", "quantile8bit", "blockwise8bit"])
def test_codec_round_trip_matches_cpu(name):
    codec = C.get_compression(name)
    n = 3 * C.QBLOCK
    x = (torch.randn(n, device=DEV, generator=_gen(8)) * 1e-2).contiguous()
    p, meta = codec.compress(x)
    out = torch.empty_like(x)
    codec.decompress_into(p, meta, out)
    pc, mc = codec.compress(x.cpu())
    outc = torch.empty(n)
    codec.decompress_into(pc, mc, outc)
    if name in ("none", "fp16", "bf16", "blockwise8bit", "quantile8bit"):
        assert torch.equal(p.cpu(), pc)                   # no reduction with a free order: identical codes
    if name in ("none", "fp16", "bf16", "blockwise8bit"):
        assert torch.equal(out.cpu(), outc)
    else:
        # means / scales are reductions whose fp32 order differs between CUDA and CPU: one code step at most
        step = float(x.abs().max()) / 100 if name != "scaled-fp16" else 1e-3 * float(x.abs().max())
        assert float((out.cpu() - outc).abs().max()) <= step


def test_blockwise_codec_rejects_partial_blocks():
    codec = C.BlockwiseQuantization()
    for n in (C.QBLOCK + 4, 100):
        with pytest.raises(ValueError, match="whole"):
            codec.compress(torch.ones(n, device=DEV))
        with pytest.raises(ValueError, match="whole"):
            codec.decompress_into(torch.zeros(n, dtype=torch.int8, device=DEV), torch.ones(1, device=DEV),
                                  torch.empty(n, device=DEV))
