"""Row-by-row oracle for the sm_90a LM-head loss kernels: the fused linear-cross-entropy of every bf16 training step
(lce_prep, lce_label_dot, the kLCEFwd GEMM epilogue, lce_finalize, the kLCEdX GEMM and the dW GEMM; csrc/lce.cu,
csrc/gemm_sm90.cu), the materialising cross-entropy on a logits tile (ce_fwd_bwd_kernel / ce_fwd_kernel) and the scoring
statistics (kLCEScore + lce_score_finalize), each against an independent float64 reference written here, fed the same
bf16 x [T, h] and W [V, h] the kernels read.

Inputs come in eight regimes, because random logits leave the softmax almost flat and the label almost never on top:
  uniform    logits ~ N(0, 1)
  peaked     logits ~ N(0, 5^2)
  confident  the label is the argmax by a gap spread over 8..30 nats across the rows: 1 - p(label) from ~1e-1 to ~1e-11
  far_label  the label sits 60..105 nats below the row maximum (inside the fused path's head-room of (100 + 58) ln 2)
  beyond     the label sits 115..150 nats below the row maximum (past the 2^100 clamp of the kLCEFwd exponent)
  zero_x     x = 0: loss = ln V and dX_t = gscale (mean_v W_v - W_y), exactly
  ignored    uniform, every 7th label is -100
  one_label  uniform, every row has the same label (the one-hot red.add of every row lands on one dW row)

The fused path is checked stage by stage: the shift c_t of lce_label_dot against z_y + 58 ln 2 (bound derived from the
fp32 dot product), the stored exponentials E element by element against exp(z - c_t) with the kernel's own c_t, the
partial row sums of every 256-column plane and the sum of squares, rowscale and the loss of lce_finalize, and dX / dW
row by row.  For dX and dW, in every tile of 64 rows (tokens for dX, vocabulary rows for dW) the worst row must stay within
``c x (the worst row of a torch bf16 materialising computation in the same tile) + floor`` (``_assert_rows``).
"""
import math

import pytest
import torch

from opendiloco_b200.models.config import LlamaConfig
from opendiloco_b200.models.llama import LlamaForCausalLM
from opendiloco_b200.ops import gemm as G
from opendiloco_b200.ops import kernels as K
from opendiloco_b200.ops import tc_gemm as TC

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
F64 = torch.float64
LN2 = math.log(2.0)
U32 = 2.0 ** -24                    # unit round-off of fp32
OFFSET = 58 * LN2                   # lce_label_dot: c_t = z_y + 58 ln 2, so the label's exponential is exactly 2^-58
CLAMP = 100.0                       # kLCEFwd: exponents (log2) are clamped at 100
REGIMES = ["uniform", "peaked", "confident", "far_label", "beyond", "zero_x", "ignored", "one_label"]
# (T, V, h): one row; a partial last 256-column plane at the 1B model's width; T not a multiple of 128; a small vocabulary
SHAPES = [(1, 32000, 1024), (127, 50264, 2048), (4161, 32000, 1024), (300, 1000, 64)]
TILE = 64
PLANE_RTOL = 1e-5                   # sum-of-squares planes against float64

# (c, floor): in every tile of 64 rows, worst row of ours <= c x worst row of the torch bf16 yardstick + floor.
# Measured on an H100 80GB HBM3 (700 W power limit), torch 2.11, over every case below: the largest ratio ours / torch
# of a tile, and the largest excess of ours over torch in a tile.
BOUND = {
    "dX": (2.0, 1e-2),             # ratio 1.87 (far_label), excess 1.5e-3; worst row 3.8e-3 (torch 2.6e-3)
    "dW": (2.0, 1e-2),             # excess 4.4e-3 (far_label, where torch's fp32 GEMM of bf16 dlogits is near exact);
                                   # ratio 8.1 (peaked, T = 1); worst row 5.0e-3 (torch 9.8e-2)
    # confident rows: p_y = 2^-58 / S, and S's label term carries the GEMM's error on z_y (~1e-5..1e-4 nats at
    # |z| ~ 30), so rowscale * E_y - gscale keeps ~1e-4 gscale |W_y| (dW: gscale |x_t|) of absolute error where
    # gscale (p_y - 1) itself may be 1e-11 gscale.  Measured: dX worst row 0.15 (T = 1), dW 0.39 (T = 127, h = 2048).
    # With the label's exponential at exp(-40) instead of 2^-58 (a 0.168% bias) the same cases measured dX 0.91..7.1
    # and dW 5.4..13.
    "dX confident": (2.0, 0.6),
    "dW confident": (2.0, 0.6),
}


# ------------------------------------------------------------------------------------------------ inputs
def _boost(x, w, rows_tok, target, measure):
    """Add a_t * w[tok_t] / |w[tok_t]|^2 to x_t so that measure(z) (fp32 logits of the bf16-rounded inputs) hits target;
    a few fixed-point steps (the boost also moves the other logits through the cross terms w_v . w_tok)."""
    u = w[rows_tok] / w[rows_tok].square().sum(1, keepdim=True)
    a = target.clone()
    wb = w.to(BF).float()
    for _ in range(8):
        z = (x + a[:, None] * u).to(BF).float() @ wb.t()
        a += target - measure(z)
    return (x + a[:, None] * u).to(BF)


def _inputs(regime, Tn, V, h, seed):
    """bf16 x [T, h], W [V, h] with |W_v| ~ 1, labels int64 [T] (distinct where the regime allows)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(Tn, h, device=DEV, generator=g)
    w = torch.randn(V, h, device=DEV, generator=g) / math.sqrt(h)
    if regime == "peaked":
        w *= 5.0
    perm = torch.randperm(V, device=DEV, generator=g)
    labels = perm[:Tn].clone()
    other = perm[Tn:2 * Tn].clone()         # every shape here has 2 T <= V
    ar = torch.arange(Tn, device=DEV)
    spread = torch.rand(Tn, device=DEV, generator=g)

    def label_gap(z):                       # z_y - max_{v != y} z_v
        zy = z[ar, labels]
        return zy - z.scatter(1, labels[:, None], float("-inf")).amax(1)

    def drop(z):                            # max_v z_v - z_y
        return z.amax(1) - z[ar, labels]

    if regime == "confident":
        xb = _boost(x, w, labels, 8.0 + 22.0 * spread, label_gap)
    elif regime in ("far_label", "beyond"):
        lo, hi = (60.0, 105.0) if regime == "far_label" else (115.0, 150.0)
        xb = _boost(x, w, other, lo + 2.0 + (hi - lo - 4.0) * spread, drop)
    else:
        xb = x.to(BF)
    if regime == "zero_x":
        xb = torch.zeros_like(xb)
    elif regime == "ignored":
        labels[::7] = -100
    elif regime == "one_label":
        labels.fill_(int(labels[0]))
    wb = w.to(BF)
    # the regime holds on the bf16 values the kernels read
    z = xb.float() @ wb.float().t()
    if regime == "confident":
        gap = label_gap(z)
        assert gap.min() > 7.5 and gap.max() < 30.5, (gap.min(), gap.max())
    elif regime in ("far_label", "beyond"):
        d = drop(z)
        assert d.min() > lo and d.max() < hi, (d.min(), d.max())
    return xb, wb, labels


# ------------------------------------------------------------------------------------------------ kernels under test
def _fused(x, w, labels, loss_scale, train=True, dw0=None):
    """Drive the kernels as LlamaEngine._head_loss_fused does.  ``labels`` are the already shifted targets: lce_prep is
    run on [0, labels...] as one sequence of T + 1 tokens, which shifts them back into place and appends the ignored
    last position."""
    Tn, h = x.shape
    V = w.shape[0]
    planes = TC.lce_planes(V)
    lab_in = torch.cat([labels.new_zeros(1), labels])
    lab = torch.empty(Tn + 1, dtype=torch.int64, device=DEV)
    n_valid, gscale, loss_sum = (torch.full((1,), float("nan"), device=DEV) for _ in range(3))
    K.lce_prep(lab_in, lab, 1, Tn + 1, loss_scale, n_valid, gscale, loss_sum)
    lab = lab[:Tn]
    sumsq = torch.zeros(1, device=DEV)
    shift = torch.full((Tn,), float("nan"), device=DEV)
    rowscale = torch.full((Tn,), float("nan"), device=DEV)
    partials = torch.full((2 * planes * Tn,), float("nan"), device=DEV)
    out = dict(labels=lab, n_valid=n_valid, gscale=gscale, loss_sum=loss_sum, sumsq=sumsq, shift=shift, partials=partials)
    K.lce_label_dot(x, w, lab, shift)
    if train:
        e = torch.full((Tn, V), float("nan"), device=DEV, dtype=BF)
        xs = torch.full((Tn, h), float("nan"), device=DEV, dtype=BF)
        dw = torch.zeros(V, h, device=DEV) if dw0 is None else dw0.clone()
        dx = torch.full((Tn, h), float("nan"), device=DEV, dtype=BF)
        TC.lce_fwd(x, w, shift, partials, e, want_sumsq=True)
        K.lce_finalize(partials, planes, lab, gscale, loss_sum, sumsq, rowscale, x, xs, dw)
        TC.lce_dx(e, w, rowscale, lab, gscale, dx)
        G.mm_tn_acc(e, xs, dw)
        out.update(e=e, xs=xs, dw=dw, dx=dx, rowscale=rowscale)
    else:
        TC.lce_fwd(x, w, shift, partials, None, want_sumsq=True)
        K.lce_finalize(partials, planes, lab, gscale, loss_sum, sumsq, None, x, None, None)
    torch.cuda.synchronize()
    return out


# ------------------------------------------------------------------------------------------------ float64 reference
def _chunk_rows(Tn, V):
    return max(1, min(Tn, (1 << 24) // V))


def _reference(x, w, labels, g, shift=None, e=None, grads=True):
    """float64 over row chunks.  Per row: z_y, lse, max_v |z_v| and sum_k |x_k w_yk| (for the rounding bounds); with
    ``grads``, dX = d W and dW = d^T x for d = g (softmax - onehot) on valid rows, and the torch bf16 yardstick of both.
    Given the kernel's shift c and exponentials E: the reference plane sums of 2^min((z - c) log2 e, 100) and of z^2,
    and the worst deviations of E."""
    Tn, h = x.shape
    V = w.shape[0]
    planes = (V + 255) // 256
    w64 = w.to(F64)
    vec = lambda: torch.empty(Tn, dtype=F64, device=DEV)                # noqa: E731
    res = dict(zy=vec(), lse=vec(), zabs=vec(), sabs=vec())
    if grads:
        res.update(dx=torch.empty(Tn, h, dtype=F64, device=DEV), dw=torch.zeros(V, h, dtype=F64, device=DEV),
                   dx_t=torch.empty(Tn, h, dtype=BF, device=DEV), dw_t=torch.zeros(V, h, device=DEV), oh_dx=vec(),
                   oh_dw=torch.zeros(V, dtype=F64, device=DEV))
    if shift is not None:
        res.update(psum=torch.empty(planes, Tn, dtype=F64, device=DEV), psq=torch.empty(planes, Tn, dtype=F64, device=DEV),
                   ptol=torch.empty(planes, Tn, dtype=F64, device=DEV),
                   e_rel=0.0, e_clamp_bad=0, e_small_max=0.0, e_clamped=0)
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False                       # the yardstick's fp32 GEMM stays fp32
    try:
        C = _chunk_rows(Tn, V)
        for c0 in range(0, Tn, C):
            c1 = min(Tn, c0 + C)
            n = c1 - c0
            xc, y = x[c0:c1], labels[c0:c1]
            valid = y >= 0
            ys = y.clamp(min=0)
            rows = torch.arange(n, device=DEV)
            x64 = xc.to(F64)
            z = x64 @ w64.t()
            res["zy"][c0:c1] = z[rows, ys]
            lse = torch.logsumexp(z, 1)
            res["lse"][c0:c1] = lse
            res["zabs"][c0:c1] = z.abs().amax(1)
            res["sabs"][c0:c1] = (x64.abs() * w64[ys].abs()).sum(1)
            if grads:
                res["oh_dx"][c0:c1] = g * w64[ys].norm(dim=1) * valid
                res["oh_dw"].index_add_(0, ys[valid], g * x64[valid].norm(dim=1))
            if shift is not None:
                cc = shift[c0:c1].to(F64)[:, None]
                arg = (z - cc) / LN2
                r = torch.exp2(arg.clamp(max=CLAMP))
                d = _exp_rtol(x64.abs() @ w64.abs().t(), z, cc, h)
                pad = planes * 256 - V
                res["psum"][:, c0:c1] = torch.nn.functional.pad(r, (0, pad)).view(n, planes, 256).sum(-1).t()
                # the plane's own fp32 sum of 256 terms: 8 further roundings at most (64 in sequence + 2 shuffles)
                res["ptol"][:, c0:c1] = torch.nn.functional.pad(r * (d + 72 * U32), (0, pad)).view(n, planes, 256).sum(-1).t()
                res["psq"][:, c0:c1] = torch.nn.functional.pad(z * z, (0, pad)).view(n, planes, 256).sum(-1).t()
                if e is not None:
                    ek = e[c0:c1].to(F64)
                    big = r >= 2.0 ** -120
                    if bool(big.any()):
                        # bf16 rounding (2^-8) plus the error of the exponent itself
                        lim = 2.0 ** -8 + d
                        rel = torch.nan_to_num((ek - r).abs() / r / lim, nan=float("inf"))
                        res["e_rel"] = max(res["e_rel"], float(rel[big].max()))
                    clamped = arg > CLAMP + 0.01
                    res["e_clamped"] += int(clamped.sum())
                    res["e_clamp_bad"] += int((clamped & (ek != 2.0 ** CLAMP)).sum())
                    if not bool(big.all()):
                        small = torch.nan_to_num(ek[~big].abs(), nan=float("inf"))
                        res["e_small_max"] = max(res["e_small_max"], float(small.max()))
                    del ek
                del arg, r, d
            if grads:
                p = torch.exp(z - lse[:, None])
                p[rows, ys] -= 1.0
                p *= g * valid[:, None]
                res["dx"][c0:c1] = p @ w64
                res["dw"] += p.t() @ x64
                del p
                # yardstick: bf16 logits, fp32 softmax - onehot, bf16 dlogits, then the two GEMMs
                lg = torch.mm(xc, w.t())
                pt = torch.softmax(lg.float(), 1)
                pt[rows, ys] -= 1.0
                dt = (pt * (g * valid[:, None])).to(BF)
                res["dx_t"][c0:c1] = torch.mm(dt, w)
                res["dw_t"] += dt.float().t() @ xc.float()
                del lg, pt, dt
            del z
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    return res


def _dot_bound(sabs, h, c):
    """|c - (z_y + 58 ln 2)| of lce_label_dot: each lane sums h / 32 products in sequence, then 5 shuffle additions and
    the offset (one more rounding at |c|), plus the fp32 representation of 58 ln 2."""
    return (h / 32 + 6) * U32 * sabs + U32 * c.abs() + 2.0 ** -19


def _exp_rtol(sabs, z, c, h):
    """Relative error of one exponential exp(z - c) of the kLCEFwd epilogue (before its bf16 rounding), from the error
    of its argument: the GEMM's fp32 accumulation of z (a recursive sum of h products bounds it by ~(h / 16 + 8) u
    sum_k |x_k w_k|; measured up to 3.6e-6 sum |x w| at h = 2048), the fp32 roundings of fma(z, log2 e, -c log2 e) and
    ex2.approx (2^-22)."""
    return (h / 16 + 8) * U32 * sabs + 4 * U32 * (z.abs() + c.abs()) + 2.0 ** -22


# ------------------------------------------------------------------------------------------------ row metric
def _row_err(x, ref, onehot):
    """|x - ref| / max(|ref|, rms / 16, 2^-12 |onehot|) per row, rms the root-mean-square row norm of ref over the tensor,
    so a row that carries almost no signal is judged on the tensor's scale instead of its own.  ``onehot`` is the size of
    the row's one-hot term (gscale |W_y| for a dX row, gscale sum |x_t| over the tokens labelled v for dW row v): the
    fused kernels add it in fp32 to a softmax term of nearly the same size, so a confidently predicted row keeps an
    absolute error of a few 1e-6 of it whatever its own size; 2^-12 of it is still 16 times below a bf16 ulp."""
    ref = ref.to(F64)
    n = ref.norm(dim=-1)
    floor = float(n.square().mean().sqrt()) / 16
    return (x.to(F64) - ref).norm(dim=-1) / torch.maximum(n.clamp_min(floor), 2.0 ** -12 * onehot)


def _tiles(err):
    pad = (-err.numel()) % TILE
    return torch.nn.functional.pad(err, (0, pad)).view(-1, TILE).amax(1)


def _check_rows(case, name, ours, theirs, ref, onehot, bound=None):
    """Worst row of ours in every tile of 64 rows <= c x the worst row of the torch bf16 yardstick in the same tile + floor.
    A reference without signal (every row ignored, or x = 0 for dW) requires ours to be exactly zero.
    Returns (summary, failure or None)."""
    if float(ref.abs().max()) == 0.0:
        ok = float(ours.float().abs().max()) == 0.0
        return f"{name} exactly 0", None if ok else f"{case}: {name} must be exactly zero"
    c, floor = BOUND[bound or name]
    e_ours, e_torch = _row_err(ours, ref, onehot), _row_err(theirs, ref, onehot)
    t_ours, t_torch = _tiles(e_ours), _tiles(e_torch)
    excess = torch.nan_to_num(t_ours - (c * t_torch + floor), nan=float("inf"))
    i = int(excess.argmax())
    pos = t_torch > 0
    ratio = float((t_ours / t_torch)[pos].max()) if bool(pos.any()) else 0.0
    need = float((t_ours - t_torch).max())
    w = int(torch.nan_to_num(e_ours, nan=float("inf")).argmax())
    line = (f"{name} worst row {float(e_ours[w]):.2e}@{w} (torch {float(e_torch.max()):.2e}), tiles <= x{ratio:.2f} torch, "
            f"excess over torch {need:.2e}")
    fail = None
    if not float(excess[i]) <= 0:
        fail = (f"{case}: {name} worst row of rows {i * TILE}..{i * TILE + TILE - 1} is {float(t_ours[i]):.3e} > {c} x torch "
                f"bf16 {float(t_torch[i]):.3e} + {floor:g} (worst row overall {float(e_ours[w]):.3e} at row {w})")
    return line, fail


# ------------------------------------------------------------------------------------------------ fused linear-cross-entropy
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "T{}-V{}-h{}".format(*s))
@pytest.mark.parametrize("regime", REGIMES)
def test_fused_lce_rows(shape, regime):
    Tn, V, h = shape
    case = f"fused T{Tn} V{V} h{h} {regime}"
    x, w, labels = _inputs(regime, Tn, V, h, 1000 * SHAPES.index(shape) + REGIMES.index(regime))
    loss_scale = 0.75
    out = _fused(x, w, labels, loss_scale)
    planes = TC.lce_planes(V)
    valid = labels >= 0
    nv = int(valid.sum())
    g = float(out["gscale"])
    ref = _reference(x, w, labels, g, out["shift"], out["e"])
    lines, failures = [case], []

    def check(ok, msg):
        if not ok:
            failures.append(f"{case}: {msg}")

    # lce_prep: shifted labels, n_valid = max(#valid, 1), gscale = loss_scale / n_valid
    check(torch.equal(out["labels"], labels), "lce_prep labels")
    check(float(out["n_valid"]) == max(nv, 1), f"n_valid {float(out['n_valid'])} != {max(nv, 1)}")
    check(abs(g - loss_scale / max(nv, 1)) <= 2 * U32 * g, f"gscale {g}")

    # lce_label_dot: c_t = z_y + 58 ln 2 within the fp32 dot-product bound ; ignored rows 0
    c = out["shift"].to(F64)
    dot_tol = _dot_bound(ref["sabs"], h, c)
    dot_err = torch.where(valid, (c - ref["zy"] - OFFSET).abs(), torch.zeros_like(c))
    i = int(torch.nan_to_num(dot_err / dot_tol, nan=float("inf")).argmax())
    lines.append(f"label_dot {float(dot_err.max()):.2e} (x{float(dot_err[i] / dot_tol[i]):.2f} of its bound)")
    check(float(dot_err[i]) <= float(dot_tol[i]), f"c_t off z_y + 58 ln 2 by {float(dot_err[i]):.3e} > {float(dot_tol[i]):.3e} at row {i}")
    check(bool((out["shift"][~valid] == 0).all()), "ignored rows: shift != 0")

    # kLCEFwd: E element by element against exp(z - c_t) with the kernel's own c_t
    lines.append(f"E x{ref['e_rel']:.4f} of its bound, {ref['e_clamped']} clamped, below 2^-120 stored <= {ref['e_small_max']:.1e}")
    check(ref["e_rel"] <= 1.0, f"E off exp(z - c) by x{ref['e_rel']:.4f} of 2^-8 + the exponent's error")
    check(ref["e_clamp_bad"] == 0, f"{ref['e_clamp_bad']} exponents above {CLAMP} are not stored as 2^{CLAMP}")
    check(ref["e_small_max"] <= 2.0 ** -118, f"an element below 2^-120 is stored as {ref['e_small_max']:.3e}")

    # partial row sums and sums of squares, per (plane, row)
    part = out["partials"].view(2, planes, Tn).to(F64)
    tiny = 256 * 2.0 ** -118
    for nm, k, r, tl in (("partial row sum", part[0], ref["psum"], ref["ptol"]),
                         ("sum of squares", part[1], ref["psq"], PLANE_RTOL * ref["psq"])):
        err = torch.nan_to_num((k - r).abs() / (tl + tiny), nan=float("inf"))
        j = int(err.argmax())
        pl, row = divmod(j, Tn)
        lines.append(f"{nm} x{float(err.view(-1)[j]):.2f} of its bound")
        check(float(err.view(-1)[j]) <= 1.0, f"{nm} of plane {pl}, row {row} off by {float((k - r).abs().view(-1)[j]):.3e} "
                                             f"> {float(tl.view(-1)[j]):.3e}")
    sq_ref = float(ref["psq"].sum())
    check(abs(float(out["sumsq"]) - sq_ref) <= PLANE_RTOL * sq_ref + tiny, f"sumsq {float(out['sumsq'])} vs {sq_ref}")

    # lce_finalize: rowscale = gscale / S, per-row loss ln S + 58 ln 2 from the kernel's partials, loss_sum
    S_k, S_r = part[0].sum(0), ref["psum"].sum(0)
    prt = (ref["ptol"].sum(0) + tiny * planes) / S_r + 2 * planes * U32          # relative error of S: planes, their fp32 sum
    rs = out["rowscale"].to(F64)
    rs_err = torch.nan_to_num(torch.where(valid, (rs - g / S_r).abs() * S_r / g / (prt + 4 * U32), rs.abs()), nan=float("inf"))
    check(float(rs_err.max()) <= 1.0, f"rowscale off by x{float(rs_err.max()):.2f} of its bound at row {int(rs_err.argmax())}")
    zero = torch.zeros_like(S_k)
    loss_k = torch.where(valid, S_k.log() + OFFSET, zero)
    loss_r = torch.where(valid, ref["lse"] - ref["zy"], zero)
    tol = torch.where(valid, dot_tol + prt + 8 * U32 * (loss_r.abs() + OFFSET), zero)
    beyond = regime == "beyond"
    if beyond:
        # the documented clamp: the row sum saturates at 2^100, the loss stays finite and below the true one
        check(bool((loss_k[valid] >= CLAMP * LN2 + OFFSET - tol[valid]).all()), "clamped loss below 100 ln 2 + 58 ln 2")
        check(bool((loss_k[valid] <= loss_r[valid] + tol[valid]).all()), "clamped loss above the float64 loss")
        check(bool(torch.isfinite(out["dx"].float()).all()) and bool(torch.isfinite(out["dw"]).all()), "non-finite gradient")
        lines.append(f"clamped row loss {float(loss_k[valid].min()):.2f}..{float(loss_k[valid].max()):.2f} "
                     f"(float64 {float(loss_r[valid].min()):.2f}..{float(loss_r[valid].max()):.2f})")
    else:
        lerr = torch.nan_to_num((loss_k - loss_r).abs(), nan=float("inf"))
        i = int((lerr / tol.clamp_min(1e-30)).argmax())
        lines.append(f"row loss {float(lerr.max()):.2e}")
        check(float(lerr[i]) <= float(tol[i]), f"row {i} loss off by {float(lerr[i]):.3e} > {float(tol[i]):.3e}")
    # lce_finalize's own arithmetic: __logf (3 ulp) and the fp32 offset per row, block sums and one atomic per 64 rows
    blocks = (Tn + 63) // 64
    order = (blocks + 8) * U32 * float(loss_k.abs().sum())
    sum_tol = Tn * 2e-5 + order
    lsum = float(out["loss_sum"])
    lines.append(f"loss_sum {lsum:.6e} (float64 {float(loss_r.sum()):.6e})")
    check(abs(lsum - float(loss_k.sum())) <= sum_tol, f"loss_sum {lsum} vs the kernel's partials {float(loss_k.sum())}")
    if not beyond:
        check(abs(lsum - float(loss_r.sum())) <= sum_tol + float(tol.sum()), f"loss_sum {lsum} vs float64 {float(loss_r.sum())}")
    # evaluation: nothing of size [T, V] is written, the statistics are bit-identical
    ev = _fused(x, w, labels, loss_scale, train=False)
    check(torch.equal(ev["partials"], out["partials"]) and torch.equal(ev["shift"], out["shift"]), "evaluation partials differ")
    if blocks == 1:
        check(torch.equal(ev["loss_sum"], out["loss_sum"]), "evaluation loss differs")
    else:                                   # one atomic per 64 rows: the order of the additions may differ
        check(abs(float(ev["loss_sum"]) - lsum) <= order, "evaluation loss differs")

    # xs = bf16(rowscale * x): the B operand of the dW GEMM
    xs_ref = out["rowscale"][:, None].to(F64) * x.to(F64)
    xs_err = (out["xs"].to(F64) - xs_ref).abs() - (2.0 ** -8 + 2.0 ** -23) * xs_ref.abs() - 2.0 ** -126
    check(bool((xs_err <= 0).all()), "xs != bf16(rowscale * x)")

    if regime == "zero_x":
        # closed forms the oracle must reproduce
        check(torch.allclose(loss_r[valid], torch.full_like(loss_r[valid], math.log(V)), rtol=0, atol=1e-12), "oracle loss != ln V")
        cf = g * (w.to(F64).mean(0)[None] - w.to(F64)[labels.clamp(min=0)]) * valid[:, None]
        check(torch.allclose(ref["dx"], cf, rtol=0, atol=1e-12 * g), "oracle dX != gscale (mean_v W_v - W_y)")
    check(int(torch.count_nonzero(out["dx"][~valid])) == 0, "ignored rows: dX != 0")
    if not beyond:
        for nm, k in (("dX", "dx"), ("dW", "dw")):
            bound = f"{nm} confident" if regime == "confident" else nm
            line, fail = _check_rows(case, nm, out[k], ref[k + "_t"], ref[k], ref["oh_" + k], bound)
            lines.append(line)
            if fail:
                failures.append(fail)
    print(" | ".join(lines))
    assert not failures, "\n".join(failures)


@pytest.mark.parametrize("shape", [(1, 32000, 1024), (300, 1000, 64)], ids=lambda s: "T{}-V{}-h{}".format(*s))
def test_fused_lce_every_row_ignored(shape):
    """No valid label: loss 0, n_valid 1, dX exactly 0 and the accumulated dW exactly unchanged."""
    Tn, V, h = shape
    x, w, labels = _inputs("uniform", Tn, V, h, 7)
    labels[:] = -100
    dw0 = torch.randn(V, h, device=DEV)
    out = _fused(x, w, labels, 1.0, dw0=dw0)
    assert float(out["n_valid"]) == 1.0 and float(out["gscale"]) == 1.0
    assert float(out["loss_sum"]) == 0.0
    assert int(torch.count_nonzero(out["dx"])) == 0
    assert torch.equal(out["dw"], dw0)
    assert bool((out["rowscale"] == 0).all()) and bool((out["shift"] == 0).all())


# ------------------------------------------------------------------------------------------------ materialising path
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "T{}-V{}-h{}".format(*s))
@pytest.mark.parametrize("regime", REGIMES)
def test_materialising_ce_elements(shape, regime):
    """ce_fwd_bwd_ (in place: dlogits) and ce_fwd on the same bf16 logits tile, element by element against float64 from
    those logits: |d - ref| <= 2^-8 (gscale p_v + |ref|) (the bf16 numerator and the bf16 result), plus 2^-120 for
    exponentials flushed to zero."""
    Tn, V, h = shape
    case = f"ce T{Tn} V{V} h{h} {regime}"
    x, w, labels = _inputs(regime, Tn, V, h, 5000 + 1000 * SHAPES.index(shape) + REGIMES.index(regime))
    logits = torch.mm(x, w.t())
    valid = labels >= 0
    nv = max(int(valid.sum()), 1)
    gscale = torch.tensor([0.75 / nv], device=DEV)
    g = float(gscale)
    d = logits.clone()
    loss_sum, sumsq, loss_f = (torch.zeros(1, device=DEV) for _ in range(3))
    K.ce_fwd_bwd_(d, labels, gscale, loss_sum, sumsq)
    K.ce_fwd(logits, labels, loss_f)
    torch.cuda.synchronize()
    worst, loss_r, loss_abs, sq_r = 0.0, 0.0, 0.0, 0.0
    C = _chunk_rows(Tn, V)
    for c0 in range(0, Tn, C):
        c1 = min(Tn, c0 + C)
        L = logits[c0:c1].to(F64)
        y = labels[c0:c1]
        ok = y >= 0
        ys = y.clamp(min=0)
        rows = torch.arange(c1 - c0, device=DEV)
        lse = torch.logsumexp(L, 1)
        rl = (lse - L[rows, ys]) * ok
        loss_r += float(rl.sum())
        loss_abs += float((lse.abs() * ok + rl.abs()).sum())
        sq_r += float((L * L).sum())
        p = torch.exp(L - lse[:, None]) * g
        ref = p.clone()
        ref[rows, ys] -= g
        ref *= ok[:, None]
        err = (d[c0:c1].to(F64) - ref).abs() / (2.0 ** -8 * (p + ref.abs()) + 2.0 ** -120)
        worst = max(worst, float(torch.nan_to_num(err, nan=float("inf")).max()))
        del L, p, ref, err
    print(f"{case} | dlogits x{worst:.2f} of the bound | loss {float(loss_sum):.6e}, ce_fwd {float(loss_f):.6e} "
          f"(float64 {loss_r:.6e})")
    assert worst <= 1.0, f"{case}: dlogits off by {worst:.3f} x the bound"
    assert int(torch.count_nonzero(d[~valid])) == 0
    # per row: __logf / ex2.approx a few ulp of lse ; the atomics add the rows in any order
    tol = Tn * 4e-6 + (Tn + 8) * U32 * loss_abs
    assert abs(float(loss_sum) - loss_r) <= tol, f"{case}: ce_fwd_bwd loss {float(loss_sum)} vs {loss_r}"
    assert abs(float(loss_f) - loss_r) <= tol, f"{case}: ce_fwd loss {float(loss_f)} vs {loss_r}"
    assert abs(float(sumsq) - sq_r) <= PLANE_RTOL * sq_r


# ------------------------------------------------------------------------------------------------ scoring statistics
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "T{}-V{}-h{}".format(*s))
@pytest.mark.parametrize("regime", ["confident", "zero_x"])
def test_score_rows(shape, regime):
    """lce_score + lce_score_finalize: lse and log p(label) per row against float64.  With x = 0 every plane ties:
    argmax = 0 and lse = ln V to within logf's one ulp."""
    Tn, V, h = shape
    case = f"score T{Tn} V{V} h{h} {regime}"
    x, w, labels = _inputs(regime, Tn, V, h, 9000 + SHAPES.index(shape))
    planes = TC.lce_planes(V)
    f32 = lambda n: torch.full((n,), float("nan"), device=DEV)           # noqa: E731
    pmax, psum, zlab = f32(planes * Tn), f32(planes * Tn), f32(Tn)
    pidx = torch.full((planes * Tn,), -1, dtype=torch.int32, device=DEV)
    TC.lce_score(x, w, labels, pmax, psum, pidx, zlab)
    lp, lse = f32(Tn), f32(Tn)
    gr = torch.zeros(Tn, dtype=torch.bool, device=DEV)
    am = torch.full((Tn,), -1, dtype=torch.int32, device=DEV)
    K.lce_score_finalize(pmax, psum, pidx, zlab, planes, labels, lp, gr, lse, am)
    torch.cuda.synchronize()
    if regime == "zero_x":
        ulp = 2.0 ** (math.floor(math.log2(math.log(V))) - 23)
        print(f"{case} | lse - ln V {float((lse.to(F64) - math.log(V)).abs().max()):.1e}")
        assert bool(((lse.to(F64) - math.log(V)).abs() <= ulp).all()), (case, lse[:4])
        assert bool((am == 0).all()) and bool((lp == -lse).all())
        assert bool(gr.eq(labels == 0).all())
        return
    ref = _reference(x, w, labels, 1.0, grads=False)
    # the label is the row maximum: z_y and lse carry the fp32 GEMM's error on the label logit, logf a few ulp of lse
    tol = 2 * (h / 32 + 6) * U32 * ref["sabs"] + 8 * U32 * ref["lse"].abs() + 1e-6
    lse_err = (lse.to(F64) - ref["lse"]).abs()
    lp_err = (lp.to(F64) - (ref["zy"] - ref["lse"])).abs()
    print(f"{case} | lse x{float((lse_err / tol).max()):.2f}, logprob x{float((lp_err / tol).max()):.2f} of the bound")
    assert bool((lse_err <= tol).all()), f"{case}: lse off by {float(lse_err.max()):.3e}"
    assert bool((lp_err <= tol).all()), f"{case}: logprob off by {float(lp_err.max()):.3e}"
    assert bool((am.long() == labels).all()) and bool(gr.all())


# ------------------------------------------------------------------------------------------------ the engine, chunked
def test_engine_head_loss_chunked(monkeypatch):
    """LlamaForCausalLM.forward_backward with T = 768 tokens over LCE chunks of 300 rows (300, 300, 168): the loss and the
    lm_head gradient rows against the oracle on the final-norm activations the engine fed its head."""
    monkeypatch.setenv("ODB_LCE_FUSED", "1")
    monkeypatch.delenv("ODB_LCE_CHUNK", raising=False)
    cfg = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4, vocab_size=3000)
    m = LlamaForCausalLM(cfg, device=DEV, seed=11, lce_chunk=300)
    ids = torch.randint(3, 3000, (3, 256), device=DEV, generator=torch.Generator(device=DEV).manual_seed(12))
    m.arena.grad.zero_()
    loss = m.forward_backward(ids, ids, 0.5)
    torch.cuda.synchronize()
    ws = next(iter(m.engine._ws.values()))
    assert ws.lce_rows == 300 and ws.T == 768 and ws._logits is None
    x, lab = ws.xnf.clone(), ws.labels.clone()
    w = m.arena.w("lm_head.weight")
    nv = int((lab >= 0).sum())
    g = float(ws.gscale)
    assert nv == 3 * 255 and abs(g - 0.5 / nv) <= 2 * U32 * g
    ref = _reference(x, w, lab, g)
    valid = lab >= 0
    loss_r = float(((ref["lse"] - ref["zy"]) * valid).sum()) / nv
    c = ref["zy"] + OFFSET
    d = _exp_rtol(ref["sabs"], ref["zabs"], c, cfg.hidden_size)           # the label's exponent: the largest |x . w| here
    tol = float((_dot_bound(ref["sabs"], cfg.hidden_size, c) + d)[valid].mean()) + 1e-5
    line, fail = _check_rows("engine", "dW", m.arena.g("lm_head.weight"), ref["dw_t"], ref["dw"], ref["oh_dw"])
    print(f"engine | loss {float(loss):.6f} (float64 {loss_r:.6f}) | {line}")
    assert fail is None, fail
    assert abs(float(loss) - loss_r) <= tol, (float(loss), loss_r)
