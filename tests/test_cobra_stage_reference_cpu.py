"""The references and checks of tests/cobra_stage_reference.py, without a GPU: each reference agrees with torch autograd in fp64, an
fp32 model of each kernel passes its check, and a model with one planted defect - a mutant of what the check guards - fails it."""
import pytest
import torch
import torch.nn.functional as F

from tests import cobra_stage_reference as sr
from tests import dense_reference as dr

LENS = [0, 1, 7, 8, 9, 17, 0, 40]          # texts without rows, at and around the 8 warps of a CTA
EPS = 1e-5


def _offsets(lens):
    o = [0]
    for n in lens:
        o.append(o[-1] + n)
    return torch.tensor(o, dtype=torch.int64)


def _seg_inputs(D, seed):
    g = torch.Generator().manual_seed(seed)
    rows = sum(LENS)
    x = torch.randn(rows, D, generator=g) * 2 + 0.5
    gam, bet = 1 + 0.1 * torch.randn(D, generator=g), 0.1 * torch.randn(D, generator=g)
    # dpooled[n] = small integers / 64 times len: dpooled / len is exact in fp32, so autograd sees the kernel's per-row gradient
    k = torch.randint(-64, 65, (len(LENS), D), generator=g).float() / 64
    dp = k * torch.tensor([max(n, 1) for n in LENS], dtype=torch.float32)[:, None]
    return x, gam, bet, dp


# ------------------------------------------------------------------------------------------------ references vs autograd
def test_seg_layernorm_mean_reference_matches_autograd():
    D = 64
    x, gam, bet, dp = _seg_inputs(D, 0)
    offs = _offsets(LENS)
    xr, gr, br = (t.double().requires_grad_(True) for t in (x, gam, bet))
    y = F.layer_norm(xr, (D,), gr, br, EPS)
    pooled = torch.stack([y[a:b].mean(0) if b > a else torch.zeros(D, dtype=torch.float64) for a, b in zip(offs[:-1], offs[1:])])
    pooled.backward(dp.double())
    f = sr.seg_layernorm_mean_forward(offs, x, gam, bet, EPS)
    assert torch.allclose(f["pooled"], pooled.detach(), rtol=1e-12, atol=1e-12)
    assert f["empty"].tolist() == [n == 0 for n in LENS]
    st = torch.stack([f["mean"], f["rstd"]], 1)
    b = sr.seg_layernorm_mean_backward(offs, x, st, gam, dp)
    for k, ref in (("dx", xr.grad), ("dg", gr.grad), ("db", br.grad)):
        assert torch.allclose(b[k], ref, rtol=1e-9, atol=1e-9), k


def test_l2norm_reference_matches_autograd():
    g = torch.Generator().manual_seed(1)
    T, D = 12, 96
    x = torch.randn(T, D, generator=g)
    x[3] = 0
    x[5] *= 1e-14                                                    # below eps: y = x / eps
    dy = torch.randn(T, D, generator=g)
    xr = x.double().requires_grad_(True)
    y = F.normalize(xr, dim=-1, eps=sr.f32(sr.L2_EPS))
    y.backward(dy.double())
    f = sr.l2norm_forward(x)
    assert torch.allclose(f["y"], y.detach(), rtol=1e-12, atol=0)
    b = sr.l2norm_backward(dy, f["y"], f["norm"])
    assert b["big"].tolist() == [i not in (3, 5) for i in range(T)]
    assert torch.allclose(b["dx"], xr.grad, rtol=1e-9, atol=0)


GROUPS = {
    "mixed": [3, 1, 4, 2],
    "one user": [7],
    "one item each": [1] * 6,
}


def _ranges(counts):
    ends = torch.tensor(counts).cumsum(0)
    user = torch.arange(len(counts)).repeat_interleave(torch.tensor(counts))
    return ends[user] - torch.tensor(counts)[user], ends[user]


@pytest.mark.parametrize("group", list(GROUPS))
def test_infonce_reference_matches_autograd(group):
    counts = GROUPS[group]
    Q = sum(counts)
    lo, hi = _ranges(counts)
    g = torch.Generator().manual_seed(2)
    S = F.normalize(torch.randn(Q, 16, generator=g), dim=-1) @ F.normalize(torch.randn(Q + 5, 16, generator=g), dim=-1).T
    S[:, Q:] = 0
    inv_tau = 4.0                                                    # a power of two: the logits are exact in fp32
    Sr = S.double().requires_grad_(True)
    keep = sr.infonce_keep(Q, lo, hi)
    logits = (Sr[:, :Q] * inv_tau).masked_fill(~keep, float("-inf"))
    rows = F.cross_entropy(logits, torch.arange(Q), reduction="none")
    rows.mean().backward()
    r = sr.infonce_rows(S, Q, lo, hi, inv_tau)
    assert torch.allclose(r["row"], rows.detach(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(r["ds"], Sr.grad, rtol=1e-12, atol=1e-14)
    assert bool(r["zero"][:, Q:].all())
    if group == "one user":
        assert bool(r["only_self"].all()) and not bool(r["row"].any())


def test_dpred_reference_matches_autograd():
    g = torch.Generator().manual_seed(3)
    Q, Qp, d = 9, 128, 32
    ds, gp, pb = torch.randn(Q, Qp, generator=g).bfloat16(), torch.randn(Qp, d, generator=g).bfloat16(), torch.randn(Q, d, generator=g).bfloat16()
    pr = pb.double().requires_grad_(True)
    (pr @ gp.double().T).backward(ds.double())
    assert torch.allclose(sr.dpred(ds, gp, pb)["dx"], pr.grad, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------ fp32 models and their mutants
def _ln_rows(x, gam, bet):
    """fp32 LayerNorm rows as ln_fwd_kernel / seg_ln_mean_fwd_kernel: two-pass mean and variance, rsqrt"""
    mean = x.mean(1, keepdim=True)
    rstd = torch.rsqrt(((x - mean) ** 2).mean(1, keepdim=True) + EPS)
    return (x - mean) * rstd * gam + bet, mean[:, 0], rstd[:, 0]


def _seg_fwd_model(offs, x, gam, bet, mutant=None):
    o = offs.tolist()
    y, mean, rstd = _ln_rows(x, gam, bet)
    out = torch.zeros(len(o) - 1, x.shape[1])
    for n in range(len(o) - 1):
        a, b = o[n], o[n + 1]
        if mutant == "last_row_skipped" and b - a > 8:
            b -= 1
        warps = [torch.zeros(x.shape[1]) for _ in range(8)]
        for r in range(a, b):
            warps[(r - a) % 8] = warps[(r - a) % 8] + y[r]
        s = torch.zeros(x.shape[1])
        for w in warps:
            s = s + w
        out[n] = s / max(o[n + 1] - a, 1)
    return out, torch.stack([mean, rstd], 1)


@pytest.mark.parametrize("mutant", [None, "last_row_skipped"])
def test_seg_layernorm_mean_forward_model_and_mutants(mutant):
    D = 192
    x, gam, bet, _ = _seg_inputs(D, 4)
    offs = _offsets(LENS)
    pooled, st = _seg_fwd_model(offs, x, gam, bet, mutant)
    f = sr.seg_layernorm_mean_forward(offs, x, gam, bet, EPS)
    ok = dr.worst(pooled, f["pooled"], f["a_pooled"]) <= dr.TOL and not bool(pooled[f["empty"]].any())
    ok = ok and dr.worst(st[:, 0], f["mean"], f["a_mean"]) <= dr.TOL and dr.worst(st[:, 1], f["rstd"], f["a_rstd"]) <= dr.TOL
    assert ok == (mutant is None), mutant


def _seg_bwd_model(offs, x, st, gam, dp, mutant=None):
    o = offs.tolist()
    D = x.shape[1]
    dx = torch.zeros_like(x)
    dg_part, db_part = [], []
    for n in range(len(o) - 1):
        a, b = o[n], o[n + 1]
        cnt = float(max(b - a, 1))
        dy = dp[n] / cnt
        warps = [torch.zeros(D) for _ in range(8)]
        for r in range(a, b):
            xh = (x[r] - st[r, 0]) * st[r, 1]
            gg = dy * gam
            sa, sb = gg.sum() / D, (gg * xh).sum() / D
            dx[r] = st[r, 1] * (gg - sa - xh * sb)
            warps[(r - a) % 8] = warps[(r - a) % 8] + dy * xh
        dg = torch.zeros(D)
        for w in warps[:7] if mutant == "dg_warp7_lost" else warps:
            dg = dg + w
        dg_part.append(dg)
        db_part.append(dy if mutant == "db_without_len" else dy * (b - a))
    return dx, torch.stack(dg_part).sum(0), torch.stack(db_part).sum(0)


@pytest.mark.parametrize("mutant", [None, "dg_warp7_lost", "db_without_len"])
def test_seg_layernorm_mean_backward_model_and_mutants(mutant):
    D = 128
    x, gam, bet, dp = _seg_inputs(D, 5)
    offs = _offsets(LENS)
    _, st = _seg_fwd_model(offs, x, gam, bet)
    dx, dg, db = _seg_bwd_model(offs, x, st, gam, dp, mutant)
    b = sr.seg_layernorm_mean_backward(offs, x, st, gam, dp)
    err = dr.errors({"dx": dx, "dg": dg, "db": db}, b, ("dx", "dg", "db"))
    assert (not dr.violations(err)) == (mutant is None), (mutant, err)


def _l2_model(x, eps, mutant=None):
    n = torch.sqrt((x * x).sum(1))
    d = n + eps if mutant == "eps_added" else n.clamp_min(eps)
    return x / d[:, None], n


def _l2_bwd_model(dy, y, n, eps, mutant=None):
    s = (dy * y).sum(1, keepdim=True)
    big = (n > eps)[:, None] if mutant != "no_eps_branch" else torch.ones_like(n, dtype=torch.bool)[:, None]
    if mutant == "no_projection":
        s = torch.zeros_like(s)
    return torch.where(big, (dy - y * s) / n[:, None].clamp_min(1e-38), dy / eps)


@pytest.mark.parametrize("mutant", [None, "eps_added", "no_eps_branch", "no_projection"])
def test_l2norm_model_and_mutants(mutant):
    g = torch.Generator().manual_seed(6)
    T, D = 10, 384
    x = torch.randn(T, D, generator=g) * 3
    x[2] = 0
    x[4] *= 3e-15                                                   # |x| ~ 6e-14 < eps
    dy = (torch.randint(-64, 65, (T, D), generator=g).float() / 64)
    eps = sr.f32(sr.L2_EPS)
    y, n = _l2_model(x, eps, mutant)
    f = sr.l2norm_forward(x)
    dx = _l2_bwd_model(dy, y, n, eps, mutant)
    b = sr.l2norm_backward(dy, y, n)
    ok = dr.worst(y, f["y"], f["a_y"]) <= dr.TOL and dr.worst(n, f["norm"], f["a_norm"]) <= dr.TOL
    ok = ok and dr.worst(dx, b["dx"], b["a_dx"]) <= dr.TOL and not bool(y[2].any())
    assert ok == (mutant is None), mutant


def _infonce_model(S, Q, lo, hi, inv_tau, mutant=None):
    """fp32 model of infonce_rows_kernel -> (row loss [Q], dS [Q, ld] bf16)"""
    ld = S.shape[1]
    l = S[:, :Q] * inv_tau
    j = torch.arange(Q)[None, :]
    i = torch.arange(Q)[:, None]
    hi_ = hi[:, None]
    keep = (j == i) | (j < lo[:, None]) | ((j > hi_) if mutant == "hi_kept_out" else (j >= hi_))
    m = l.masked_fill(~keep, float("-inf")).amax(1, keepdim=True)
    e = torch.where(keep, torch.exp(l - m), torch.zeros_like(l))
    z = e.sum(1, keepdim=True)
    row = torch.log(z[:, 0]) + m[:, 0] - torch.diagonal(l)
    gs = torch.tensor(inv_tau, dtype=torch.float32) / (Q - 1 if mutant == "gscale_q_minus_1" else Q)
    g = torch.where(keep, (e * (1 / z) - (j == i).float()) * gs, torch.zeros_like(l))
    ds = torch.zeros(Q, ld)
    ds[:, :Q] = g
    return row, ds.bfloat16()


@pytest.mark.parametrize("mutant", [None, "gscale_q_minus_1", "hi_kept_out"])
def test_infonce_model_and_mutants(mutant):
    """users of 3, 1, 4 and 2 items at Q = 10, padded to 128 columns, tau = 0.2 (an inv_tau whose products round)"""
    counts = GROUPS["mixed"]
    Q = sum(counts)
    lo, hi = _ranges(counts)
    g = torch.Generator().manual_seed(7)
    S = torch.zeros(Q, 128)
    S[:, :Q] = F.normalize(torch.randn(Q, 32, generator=g), dim=-1) @ F.normalize(torch.randn(Q, 32, generator=g), dim=-1).T
    row, ds = _infonce_model(S, Q, lo, hi, 1 / 0.2, mutant)
    r = sr.infonce_rows(S, Q, lo, hi, 1 / 0.2)
    ok = dr.worst(row, r["row"], r["a_row"]) <= dr.TOL and dr.worst(ds, r["ds"], r["a_ds"]) <= dr.TOL
    ok = ok and not bool(ds[r["zero"]].any())
    assert ok == (mutant is None), mutant
