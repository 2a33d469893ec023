"""fp64 references of COBRA's own kernels (csrc/cobra.cuh) - the pooled LayerNorm mean over each text, the L2 normalisation and
the in-batch InfoNCE rows - and of the dpred GEMM that follows them, in the style of tests/dense_reference.py: each takes the kernel's
own inputs (and, for a backward, what its forward saved), computes in exact fp64 and returns a per-element allowance for the
kernel's rounding.  A check divides the error by the allowance (dense_reference.worst) and holds it to dense_reference.TOL = 1.

Where the kernels round (C = 2^-24 the fp32 unit roundoff, U = 2^-8 half a bf16 ulp, both relative):
  pooled LayerNorm mean   seg_ln_mean_fwd_kernel: each row's LayerNorm as ln_fwd_kernel (dense_reference.layernorm_forward,
                          a_y32), then warp w of the text's CTA sums rows w, w + 8, ... in order and the 8 warp sums are added in
                          order (ceil(len / 8) + 8 terms deep), then one correctly rounded division by len.  A text without rows
                          pools to exactly 0.
  its backward            seg_ln_mean_bwd_kernel: every row of text n takes dy = fp32(dpooled[n] / len) (restated exactly here),
                          then the LayerNorm backward from the saved stats (dense_reference.layernorm_backward).  dg: the per-warp,
                          per-text and then det_finish's over-texts sums; db: fp32(dpooled[n] / len) * len per text (two
                          roundings), then the over-texts sum.  A text without rows adds exactly 0 to both.
  L2 norm                 l2norm_fwd_kernel: n = sqrtf(sum x^2) (fmaf per lane, D / 32 terms, then a 5-level butterfly; sqrtf is
                          the approximate one under --use_fast_math, DIV), y = x / max(n, eps) correctly rounded.  Squares below
                          2^-126 flush to zero, so the norm has an absolute floor.
  its backward            l2norm_bwd_kernel from the saved (y, n): where n > eps, dx = (dy - y (dy . y)) / n, the dot product as
                          the forward's sum; else dx = dy / eps, one rounding.
  InfoNCE rows            infonce_rows_kernel on the fp32 scores S: the logits fp32(S inv_tau) (restated exactly here), their max
                          over the kept columns, z = sum exp_accurate(l - m) (256 threads, Q / 256 terms each, a butterfly, 8 warp
                          sums in order), row_loss = logf(z) + m - l_ii; dS = bf16((exp_accurate(l - m) fp32(1 / z) - [i == j])
                          fp32(inv_tau / Q)).  The left-out columns [lo, hi) other than i and the padding columns [Q, ld) hold an
                          exact 0; a row that keeps only itself has z = exp_accurate(0) = 1 and a row loss of exactly 0.
  dpred                   the wgmma GEMM dS gpad, fp32: dense_reference.linear_backward on the kernel's bf16 dS.
"""
import math

import torch

from tests import dense_reference as dr
from tests.attention_reference import U

C = dr.C
ACC = dr.ACC
DIV = 2.0 ** -21               # approximate sqrtf / logf under --use_fast_math: 4 ulp
EXP = 2.0 ** -20               # exp_accurate: degree-6 polynomial on |r| <= ln2 / 2 plus its fmaf chain, relative
LOG = 2.0 ** -20               # __logf on z in [1, Q]: absolute
L2_EPS = 1e-12                 # F.normalize


def f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _offsets(offsets):
    o = [int(v) for v in offsets.tolist()]
    return o, [b - a for a, b in zip(o, o[1:])]


# ------------------------------------------------------------------------------------------------ pooled LayerNorm mean
def seg_layernorm_mean_forward(offsets, x, g, b, eps):
    """offsets [N + 1], x [rows, D] fp32.  -> "pooled" [N, D] with "a_pooled", "mean" / "rstd" [rows] with "a_mean" / "a_rstd"
    (one entry per row, as the kernel's stats), "empty" [N] bool (texts without rows: pooled exactly 0)."""
    o, lens = _offsets(offsets)
    N, D = len(lens), g.numel()
    dev = x.device
    pooled = torch.zeros(N, D, dtype=torch.float64, device=dev)
    allow = torch.zeros(N, D, dtype=torch.float64, device=dev)
    r = {"pooled": pooled, "a_pooled": allow, "empty": torch.tensor([n == 0 for n in lens], device=dev)}
    if o[-1] == 0:
        empty = torch.zeros(0, dtype=torch.float64, device=dev)
        return {**r, "mean": empty, "a_mean": empty, "rstd": empty, "a_rstd": empty}
    ln = dr.layernorm_forward(x[:o[-1]], g, b, eps)
    for n in range(N):
        if lens[n] == 0:
            continue
        y, a = ln["y"][o[n]:o[n + 1]], ln["a_y32"][o[n]:o[n + 1]]
        depth = -(-lens[n] // 8) + 8
        pooled[n] = y.sum(0) / lens[n]
        allow[n] = (a.sum(0) + depth * C * y.abs().sum(0)) / lens[n] + C * pooled[n].abs()
    return {**r, **{k: ln[k] for k in ("mean", "a_mean", "rstd", "a_rstd")}}


def seg_layernorm_mean_backward(offsets, x, stats, g, dpooled):
    """From the kernel's saved stats [rows, 2].  -> "dx" [rows, D], "dg", "db" [D] with allowances, "dy" [rows, D] fp32 (the per-row
    gradient fp32(dpooled[n] / len) the kernel feeds its LayerNorm backward)."""
    o, lens = _offsets(offsets)
    N, D = len(lens), g.numel()
    dev = x.device
    cnt = torch.tensor([max(n, 1) for n in lens], dtype=torch.float32, device=dev)
    dyt = dpooled.float() / cnt[:, None]                                       # __fdiv_rn, exactly
    live = torch.tensor(lens, device=dev) > 0
    DP = dpooled.double()
    db = DP[live].sum(0)
    a_db = 2 * C * DP[live].abs().sum(0) + (N + 2) * ACC * DP[live].abs().sum(0)
    rows = o[-1]
    if rows == 0:
        z = torch.zeros(0, D, dtype=torch.float64, device=dev)
        zd = torch.zeros(D, dtype=torch.float64, device=dev)
        return {"dx": z, "a_dx": z, "dg": zd, "a_dg": zd, "db": db, "a_db": a_db, "dy": z.float()}
    text = torch.repeat_interleave(torch.arange(N, device=dev), torch.tensor(lens, device=dev))
    dy = dyt[text]
    lb = dr.layernorm_backward(dy, x[:rows], stats[:rows], g)
    X, st = x[:rows].double(), stats[:rows].double()
    xh = (X - st[:, 0:1]) * st[:, 1:2]
    e_xh = 2 * C * (xh.abs() + st[:, 1:2] * X.abs())
    depth = -(-max(lens) // 8) + 8 + N + 2
    a_dg = depth * ACC * (dy.double().abs() * (xh.abs() + e_xh)).sum(0)
    return {"dx": lb["dx"], "a_dx": lb["a_dx"], "dg": lb["dg"], "a_dg": a_dg, "db": db, "a_db": a_db, "dy": dy}


# ------------------------------------------------------------------------------------------------ L2 norm
def l2norm_forward(x, eps=L2_EPS):
    """x [T, D] fp32.  -> "y" with "a_y", "norm" [T] with "a_norm"."""
    X = x.double()
    D = X.shape[1]
    n = X.norm(dim=1)
    e_n = (D // 32 + 6) * C / 2 + DIV                                          # relative
    a_n = e_n * n + 2.0 ** -63 * math.sqrt(D)                                  # FTZ of squares below 2^-126
    d = n.clamp_min(f32(eps))
    y = X / d[:, None]
    big = n > f32(eps)
    rel = torch.where(big, e_n + C + 2.0 ** -63 * math.sqrt(D) / n.clamp_min(1e-300), torch.full_like(n, C))
    return {"y": y, "a_y": y.abs() * rel[:, None] + 2.0 ** -149, "norm": n, "a_norm": a_n}


def l2norm_backward(dy, y, norm, eps=L2_EPS):
    """From the kernel's saved (y [T, D], norm [T]).  -> "dx" with "a_dx", "big" [T] (the rows of the n > eps branch)."""
    DY, Y, n = dy.double(), y.double(), norm.double()
    D = Y.shape[1]
    big = norm.float() > f32(eps)
    s = (DY * Y).sum(1, keepdim=True)
    a_s = (D // 32 + 6) * C * (DY * Y).abs().sum(1, keepdim=True)
    nn_ = n[:, None].clamp_min(1e-300)
    dx_big = (DY - Y * s) / nn_
    a_big = (Y.abs() * a_s + 2 * C * (DY.abs() + (Y * s).abs())) / nn_ + C * dx_big.abs()
    dx_small = DY / f32(eps)
    dx = torch.where(big[:, None], dx_big, dx_small)
    a_dx = torch.where(big[:, None], a_big, C * dx_small.abs())
    return {"dx": dx, "a_dx": a_dx, "big": big}


# ------------------------------------------------------------------------------------------------ InfoNCE
def infonce_keep(Q, lo, hi, device="cpu"):
    """[Q, Q] bool: the columns row i takes part in - outside [lo[i], hi[i]), plus i itself"""
    j = torch.arange(Q, device=device)[None, :]
    i = torch.arange(Q, device=device)[:, None]
    return (j == i) | (j < lo.to(device)[:, None]) | (j >= hi.to(device)[:, None])


def infonce_rows(S, Q, lo, hi, inv_tau):
    """S [Q, ld] fp32 (the kernel's own scores; columns [Q, ld) are padding), lo / hi [Q].  -> "row" [Q] with "a_row", "loss" (their
    mean) with "a_loss", "ds" [Q, ld] with "a_ds" (the fp64 value of (softmax - delta) / (Q tau)), "keep" [Q, Q], "zero" [Q, ld]
    bool (the cells dS must hold an exact 0), "only_self" [Q] bool (rows whose loss must be exactly 0)."""
    dev = S.device
    ld = S.shape[1]
    it = f32(inv_tau)
    l = (S[:, :Q].float() * it).double()                                       # the kernel's fp32 logits, exactly
    keep = infonce_keep(Q, lo, hi, dev)
    lm = l.masked_fill(~keep, float("-inf"))
    m = lm.amax(1, keepdim=True)
    e = torch.exp(lm - m)
    z = e.sum(1, keepdim=True)
    P = e / z
    diag = torch.diagonal(l)
    row = torch.log(z[:, 0]) + m[:, 0] - diag
    # relative error of each exp term (the rounded difference l - m, exp_accurate) and of z (the Q / 256 + 13 deep fp32 sum)
    e_term = torch.where(keep, EXP + C * (l - m).abs(), torch.zeros_like(l))
    e_z = (e * e_term).sum(1) / z[:, 0] + (Q // 256 + 13) * C
    a_row = e_z + LOG + 2 * C * (torch.log(z[:, 0]).abs() + m[:, 0].abs() + diag.abs() + row.abs())
    eye = torch.eye(Q, dtype=torch.float64, device=dev)
    gs = it / Q
    ds = torch.zeros(Q, ld, dtype=torch.float64, device=dev)
    ds[:, :Q] = torch.where(keep, (P - eye) * gs, torch.zeros_like(P))
    e_p = (e_term + e_z[:, None] + 2 * C) * P                                  # absolute error of the fp32 probability
    a_ds = torch.zeros_like(ds)
    a_ds[:, :Q] = torch.where(keep, U * ds[:, :Q].abs() + (1 + U) * (e_p * gs + 3 * C * ds[:, :Q].abs()), torch.zeros_like(P))
    zero = torch.ones(Q, ld, dtype=torch.bool, device=dev)
    zero[:, :Q] = ~keep
    only_self = keep.sum(1) == 1
    loss = row.mean()
    a_loss = (a_row.sum() + Q * ACC * row.abs().sum()) / Q + C * loss.abs()
    return {"row": row, "a_row": a_row, "loss": loss, "a_loss": a_loss, "ds": ds, "a_ds": a_ds, "keep": keep, "zero": zero,
            "only_self": only_self}


def dpred(ds, gpad, pred_b):
    """the dpred GEMM on the kernel's bf16 dS [Q, Qp] and gpad [Qp, d] -> "dx" [Q, d] with "a_dx" (dense_reference.linear_backward)"""
    return dr.linear_backward(ds, gpad, pred_b)
