"""One-shot drivers for `ncu --set full` captures of individual kernels at the Llama-150M micro-batch shapes.

    ncu --set full --clock-control none --import-source on -k regex:<kernel> -s 2 -c 1 -o profiles_out/<name> \
        python profiles/ncu_one.py <which>

which: lce | bandwidth (AdamW, grad norm, RMSNorm fwd/bwd, embedding fwd/bwd, LCE helpers, Nesterov solo, cast)
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from opendiloco_b200.ops import gemm as G  # noqa: E402
from opendiloco_b200.ops import kernels as K  # noqa: E402
from opendiloco_b200.ops import tc_gemm as T  # noqa: E402

which = sys.argv[1] if len(sys.argv) > 1 else "lce"
BF, dev = torch.bfloat16, "cuda"
Tn, V, h, P = 32768, 32000, 1024, 214_990_848
torch.manual_seed(0)
REPS = 3

if which == "lce":
    x = torch.randn(Tn, h, device=dev).to(BF)
    w = (torch.randn(V, h, device=dev) * 0.02).to(BF)
    labels = torch.randint(0, V, (Tn,), device=dev)
    gscale = torch.full((1,), 1.0 / Tn, device=dev)
    loss_sum = torch.zeros(1, device=dev)
    planes = T.lce_planes(V)
    shift, rowscale = torch.empty(Tn, device=dev), torch.empty(Tn, device=dev)
    partials = torch.empty(2 * planes * Tn, device=dev)
    e = torch.empty(Tn, V, device=dev, dtype=BF)
    xs = torch.empty(Tn, h, device=dev, dtype=BF)
    dw = torch.zeros(V, h, device=dev)
    dx = torch.empty(Tn, h, device=dev, dtype=BF)
    for _ in range(REPS):
        K.lce_label_dot(x, w, labels, shift)
        T.lce_fwd(x, w, shift, partials, e)
        K.lce_finalize(partials, planes, labels, gscale, loss_sum, None, rowscale, x, xs, dw)
        T.lce_dx(e, w, rowscale, labels, gscale, dx)
        G.mm_tn_acc(e, xs, dw)
elif which == "bandwidth":
    n = P
    p, g, m, v = (torch.randn(n, device=dev) * 0.02 for _ in range(4))
    v.abs_()
    shadow = torch.empty(n, device=dev, dtype=BF)
    hp = torch.zeros(K.HP_SIZE, device=dev)
    hp[K.HP_LR], hp[K.HP_B1], hp[K.HP_B2], hp[K.HP_EPS], hp[K.HP_WD] = 4e-4, 0.9, 0.95, 1e-8, 0.1
    hp[K.HP_BC1], hp[K.HP_BC2], hp[K.HP_MAXNORM], hp[K.HP_INVSCALE] = 0.1, 0.05, 1.0, 1.0
    partials = torch.zeros(K.MAX_PARTIALS, device=dev)
    flag = torch.zeros(1, dtype=torch.int32, device=dev)
    stats = torch.zeros(2, device=dev)
    theta_outer, buf = p.clone(), torch.zeros(n, device=dev)
    xa = torch.randn(Tn, h, device=dev).to(BF)
    delta = torch.randn(Tn, h, device=dev).to(BF)
    wn = torch.ones(h, device=dev, dtype=BF)
    y, xo = torch.empty_like(xa), torch.empty_like(xa)
    rstd = torch.empty(Tn, device=dev)
    dwn = torch.zeros(h, device=dev)
    dres = torch.empty_like(xa)
    ids = torch.randint(0, V, (Tn,), device=dev)
    emb = (torch.randn(V, h, device=dev) * 0.02).to(BF)
    demb = torch.zeros(V, h, device=dev)
    for _ in range(REPS):
        npart = K.grad_sqnorm(g, partials, flag)
        K.adamw_step(p, g, m, v, shadow, hp, partials, npart, None, stats, zero_grad=True)
        K.nesterov_outer(theta_outer, buf, None, p, shadow, 0.7, 0.9, True)
        K.rmsnorm_fwd(xa, wn, 1e-5, delta=delta, out=y, rstd=rstd, x_out=xo)
        K.rmsnorm_bwd(y, xo, wn, rstd, delta, dres, dwn)
        K.embedding_fwd(ids, emb, out=y)
        K.embedding_bwd(ids, y, demb)
        K.cast_to_bf16(p, shadow)
torch.cuda.synchronize()
