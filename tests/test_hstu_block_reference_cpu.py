"""The references and checks of tests/hstu_block_reference.py, without a GPU: each reference agrees with torch autograd in fp64, an
fp32 model of each kernel (ln_gate_fwd, ln_gate_bwd, cast_colsum, the HSTU attention with its 64-key tiles and bf16 packs, the Adam
step) passes its check at the GPU tolerance, and a model with one planted defect - a mutant of what the check guards - fails it."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import dense_reference as dr
from tests import hstu_block_reference as hr

EPS = hr.EPS


def _ok(items):
    """True when every (got, ref, allowance) is within dense_reference.TOL"""
    return all(dr.worst(g, r, a) <= dr.TOL for g, r, a in items)


def _gate_inputs(T, D, seed):
    """bf16 O with a zero row and large row offsets (for LN1), bf16 U and zu, fp32 x with +-1000 offsets on every third row"""
    g = torch.Generator().manual_seed(seed)
    O = torch.randn(T, D, generator=g)
    O[1::4] += torch.tensor([100.0, -300.0, 700.0]).repeat(T)[: O[1::4].shape[0], None]
    O[0] = 0
    zu = (1.5 * torch.randn(T, D, generator=g)).bfloat16()
    U = F.silu(zu.float()).bfloat16()
    x = torch.randn(T, D, generator=g)
    x[::3] += 1000.0
    prm = dict(g1=1 + 0.1 * torch.randn(D, generator=g), b1=0.1 * torch.randn(D, generator=g) + 0.5,
               g2=1 + 0.1 * torch.randn(D, generator=g), b2=0.1 * torch.randn(D, generator=g))
    return O.bfloat16(), U, zu, x, prm


def _ln_stats(v, one_pass=False):
    mean = v.mean(1, keepdim=True)
    var = (v * v).mean(1, keepdim=True) - mean * mean if one_pass else ((v - mean) ** 2).mean(1, keepdim=True)
    return mean, torch.rsqrt(var + EPS)


# ------------------------------------------------------------------------------------------------ references vs autograd
def test_gate_reference_matches_autograd():
    T, D, p, seed, site = 9, 64, 0.5, 3, 8
    O, U, zu, x, prm = _gate_inputs(T, D, 0)
    Or, zr, xr = O.double().requires_grad_(True), zu.double().requires_grad_(True), x.double().requires_grad_(True)
    pr = {k: v.double().requires_grad_(True) for k, v in prm.items()}
    km = dr.keep(range(T), D, p, seed, site)
    x1 = xr + F.layer_norm(Or, (D,), pr["g1"], pr["b1"], EPS) * F.silu(zr) * km
    x1.retain_grad()
    xn = F.layer_norm(x1, (D,), pr["g2"], pr["b2"], EPS)
    g = torch.Generator().manual_seed(1)
    dy, dxn = torch.randn(T, D, generator=g), torch.randn(T, D, generator=g)
    (x1 * dy.double()).sum().add((xn * dxn.double()).sum()).backward()
    f = hr.gate_forward(O, F.silu(zu.double()), x, x1.detach(), prm["g1"], prm["b1"], prm["g2"], prm["b2"], p, seed, site)
    assert torch.allclose(f["x1"], x1.detach(), rtol=1e-10, atol=1e-10)
    assert torch.allclose(f["xn"], xn.detach(), rtol=1e-9, atol=1e-9)
    st = lambda m, r: torch.stack([m, r], 1)                              # noqa: E731
    b = hr.gate_backward(dy, dxn, x1.detach(), st(f["mean1"], f["rstd1"]), st(f["mean2"], f["rstd2"]), O, F.silu(zu.double()), zu,
                         x1.grad, prm["g1"], prm["b1"], prm["g2"], p, seed, site)
    for k, ref in (("dx1", x1.grad), ("dzu", zr.grad), ("dO", Or.grad), ("dg1", pr["g1"].grad), ("db1", pr["b1"].grad),
                   ("dg2", pr["g2"].grad), ("db2", pr["b2"].grad)):
        assert torch.allclose(b[k], ref, rtol=1e-8, atol=1e-8), k


def test_block_stage_references_match_autograd():
    """cast_colsum (db of the FFN output) and linear_dact_backward against autograd of the FFN's second half"""
    g = torch.Generator().manual_seed(2)
    T, D, p, seed, site = 11, 16, 0.5, 4, 2
    dy = torch.randint(-64, 65, (T, D), generator=g).float() / 64
    cc = hr.cast_colsum(dy, p, seed, site)
    km = dr.keep(range(T), D, p, seed, site)
    b = torch.zeros(D, dtype=torch.float64, requires_grad=True)
    ((torch.zeros(T, D, dtype=torch.float64) + b) * km).mul(dy.double()).sum().backward()
    assert torch.equal(cc["db"], b.grad)
    assert torch.equal(cc["dyb_exact"].double(), (dy.double() * km))
    z = torch.randn(T, 4 * D, generator=g).bfloat16()
    w = (0.1 * torch.randn(D, 4 * D, generator=g)).bfloat16()
    zr = z.double().requires_grad_(True)
    kh = dr.keep(range(T), 4 * D, p, seed, site - 1)
    h = F.silu(zr) * kh
    h.backward(cc["dyb_exact"].double() @ w.double())
    assert torch.allclose(hr.linear_dact_backward(cc["dyb_exact"], w, z, p, seed, site - 1)["g"], zr.grad, rtol=1e-12, atol=1e-12)


def _attn_inputs(B, L, D, H, npos=8, nt=20, seed=0):
    """bf16 zp, P = silu(zp), dO, a pad pattern (mid pad, left pad, fully padded row), an index matrix of random buckets, tables"""
    g = torch.Generator().manual_seed(seed)
    zp = (0.7 * torch.randn(B, L, 4 * D, generator=g)).bfloat16()
    P = F.silu(zp.float()).bfloat16()
    dO = (torch.randn(B, L, D, generator=g) / max(1.0, L ** 0.5)).bfloat16()
    pad = torch.zeros(B, L, dtype=torch.bool)
    pad[0, L // 2] = True
    pad[1, : L // 3] = True
    if B > 2:
        pad[2] = True
    ii = torch.arange(L)
    pb = torch.randint(0, npos, (L,), generator=g)[(ii[:, None] - ii[None, :]).clamp_min(0)]
    tb = torch.randint(0, nt, (B, L, L), generator=g)
    valid = hr.causal_valid(pad)[:, 0]
    idx = torch.where(valid, pb[None] * 64 + tb, torch.full_like(tb, npos * 64)).to(torch.int16)
    wpos, wtime = 0.3 * torch.randn(npos, H, generator=g), 0.5 * torch.randn(nt, H, generator=g)
    w, masked, _, _ = hr.cell_bias(idx, wpos, wtime, npos, H)
    assert torch.equal(masked[:, 0], ~valid)
    return zp, P, dO, pad, w


def test_attention_reference_matches_autograd():
    B, L, D, H = 3, 21, 32, 2
    zp, P, dO, pad, w = _attn_inputs(B, L, D, H)
    zr = zp.double().requires_grad_(True)
    Pf = F.silu(zr)
    Pq = Pf + (P.double() - Pf).detach()                 # forward on the bf16 activations, backward through silu(zp)
    _, V, Q, K = Pq.chunk(4, -1)
    hs = lambda t: t.reshape(B, L, H, D // H).transpose(1, 2)              # noqa: E731
    S = hs(Q) @ hs(K).transpose(-1, -2) + w.double()
    S.retain_grad()
    valid = hr.causal_valid(pad)
    O = (torch.where(valid, F.silu(S), torch.zeros_like(S)) @ hs(V)).transpose(1, 2).reshape(B, L, D)
    O.backward(dO.double())
    r = hr.attention(P, w, valid, H, zp, dO)
    assert torch.allclose(r["O"], O.detach(), rtol=1e-10, atol=1e-12)
    assert torch.allclose(r["dS"], torch.where(valid, S.grad, torch.zeros_like(S)), rtol=1e-10, atol=1e-12)
    for name, lo in (("dV", D), ("dQ", 2 * D), ("dK", 3 * D)):
        assert torch.allclose(r[name], zr.grad[..., lo:lo + D], rtol=1e-10, atol=1e-12), name


@pytest.mark.parametrize("t", [1, 2, 10, 1000])
def test_adam_reference_matches_torch(t):
    g = torch.Generator().manual_seed(t)
    n = 100
    p0, g0 = torch.randn(n, generator=g).double(), torch.randn(n, generator=g).double()
    m0, v0 = 1e-2 * torch.randn(n, generator=g).double(), 1e-3 * torch.rand(n, generator=g).double()
    hyp = dict(lr=hr.f32(1e-3), betas=(hr.f32(0.9), hr.f32(0.999)), eps=hr.f32(1e-8), weight_decay=hr.f32(1e-2))
    q = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([q], **hyp)
    q.grad = g0 * 0.125
    opt.state[q] = {"step": torch.tensor(float(t - 1), dtype=torch.float64), "exp_avg": m0.clone(), "exp_avg_sq": v0.clone()}
    opt.step()
    r = hr.adam(p0, g0, m0, v0, t, 1e-3, 0.9, 0.999, 1e-8, 1e-2, 0.125)
    assert torch.allclose(r["p"], q.detach(), rtol=1e-12, atol=1e-14)
    assert torch.allclose(r["m"], opt.state[q]["exp_avg"], rtol=1e-12, atol=1e-16)
    assert torch.allclose(r["v"], opt.state[q]["exp_avg_sq"], rtol=1e-12, atol=1e-18)


# ------------------------------------------------------------------------------------------------ gate models and mutants
def gate_fwd_model(O, Uc, x, prm, p, seed, site, mutant=None):
    """fp32 model of ln_gate_fwd_kernel -> x1, xn (bf16), st1, st2; a skipped row keeps the NaN the buffers start with"""
    T, D = O.shape
    o, u = O.float(), Uc.float()
    m1, r1 = _ln_stats(o, mutant == "one_pass_var")
    n = (o - m1) * r1 * prm["g1"] + (0 if mutant == "no_b1" else prm["b1"])
    rows = np.arange(T) + (1 if mutant == "gate_row_key" else 0)
    km = dr.keep(rows, D, p, seed, site + (1 if mutant == "gate_site" else 0)).float()
    if mutant == "no_keep_scale":
        km = (km != 0).float()
    x1 = x + n * u * km
    m2, r2 = _ln_stats(x if mutant == "xn_from_x" else x1)
    xn = ((x if mutant == "xn_from_x" else x1) - m2) * r2 * prm["g2"] + prm["b2"]
    out = dict(x1=x1, xn=xn.bfloat16(), st1=torch.cat([m1, r1], 1), st2=torch.cat([m2, r2], 1))
    if mutant == "skip_last_row_fwd":
        for k in out:
            out[k][-1] = float("nan")
    return out


def gate_bwd_model(dy, dxn, f, O, Uc, zu, prm, p, seed, site, mutant=None):
    """fp32 model of ln_gate_bwd_kernel (the parameter sums in plain fp32) -> dx1, dzu (bf16), dO (bf16), dg1, db1, dg2, db2"""
    T, D = O.shape
    x1, st1, st2 = f["x1"], f["st1"], f["st2"]
    live = torch.ones(T, 1)
    if mutant == "skip_last_row_bwd":
        live[-1] = 0
    m2, r2 = st2[:, 0:1], st2[:, 1:2]
    xh2 = (x1 - m2) * r2
    gg = dxn * prm["g2"]
    dx1 = (0 if mutant == "no_dy_residual" else dy) + r2 * (gg - gg.mean(1, keepdim=True) - xh2 * (gg * xh2).mean(1, keepdim=True))
    km = dr.keep(range(T), D, p, seed, site).float()
    dG = dx1 if mutant == "no_drop_dG" else dx1 * km
    m1, r1 = st1[:, 0:1], st1[:, 1:2]
    o, u, z = O.float(), Uc.float(), zu.float()
    xh1 = (o - m1) * r1
    n = xh1 * prm["g1"] + prm["b1"]
    ds = {"dzu_no_dsilu": torch.ones_like(z), "dzu_dsilu_U": hr.dsilu(u)}.get(mutant, hr.dsilu(z))
    dzu = dG * n * ds
    dN = dG if mutant == "dO_no_U" else dG * u
    gn = dN * prm["g1"]
    dO = r1 * (gn - gn.mean(1, keepdim=True) - xh1 * (gn * xh1).mean(1, keepdim=True))
    dN1 = dx1 * u if mutant == "dg1_undropped" else dN
    out = dict(dx1=dx1, dzu=dzu.bfloat16(), dO=dO.bfloat16(), dg1=(live * dN1 * xh1).sum(0), db1=(live * dN).sum(0),
               dg2=(live * dxn * xh2).sum(0), db2=(live * dxn).sum(0))
    if mutant == "skip_last_row_bwd":
        for k in ("dx1", "dzu", "dO"):
            out[k][-1] = float("nan")
    return out


GATE_FWD_MUTANTS = ["gate_site", "gate_row_key", "no_keep_scale", "one_pass_var", "no_b1", "xn_from_x", "skip_last_row_fwd"]
GATE_BWD_MUTANTS = ["no_drop_dG", "dzu_no_dsilu", "dzu_dsilu_U", "dO_no_U", "dg1_undropped", "no_dy_residual", "skip_last_row_bwd"]


def _gate_check(O, U, zu, x, prm, dy, dxn, p, seed, site, fwd_mut, bwd_mut):
    f = gate_fwd_model(O, U, x, prm, p, seed, site, fwd_mut)
    rf = hr.gate_forward(O, U, x, f["x1"], prm["g1"], prm["b1"], prm["g2"], prm["b2"], p, seed, site)
    ok = _ok([(f["x1"], rf["x1"], rf["a_x1"]), (f["xn"], rf["xn"], rf["a_xn"]), (f["st1"][:, 0], rf["mean1"], rf["a_mean1"]),
              (f["st1"][:, 1], rf["rstd1"], rf["a_rstd1"]), (f["st2"][:, 0], rf["mean2"], rf["a_mean2"]),
              (f["st2"][:, 1], rf["rstd2"], rf["a_rstd2"])])
    ok = ok and not bool((f["x1"] - x)[rf["drop"]].any())
    if fwd_mut is not None:
        return ok
    b = gate_bwd_model(dy, dxn, f, O, U, zu, prm, p, seed, site, bwd_mut)
    rb = hr.gate_backward(dy, dxn, f["x1"], f["st1"], f["st2"], O, U, zu, b["dx1"], prm["g1"], prm["b1"], prm["g2"], p, seed, site)
    return ok and _ok([(b[k], rb[k], rb["a_" + k]) for k in ("dx1", "dzu", "dO", "dg1", "db1", "dg2", "db2")])


@pytest.mark.parametrize("mutant", [None] + GATE_FWD_MUTANTS + GATE_BWD_MUTANTS)
def test_gate_model_and_mutants(mutant):
    T, D, seed, site = 97, 128, 5, 24
    O, U, zu, x, prm = _gate_inputs(T, D, 1)
    g = torch.Generator().manual_seed(3)
    dy, dxn = torch.randint(-64, 65, (T, D), generator=g).float() / 64, torch.randn(T, D, generator=g)
    fwd = mutant if mutant in GATE_FWD_MUTANTS else None
    bwd = mutant if mutant in GATE_BWD_MUTANTS else None
    oks = [_gate_check(O, U, zu, x, prm, dy, dxn, p, seed, site, fwd, bwd) for p in (0.0, 0.2, 0.5)]
    if mutant is None:
        assert all(oks), oks
    else:
        assert not all(oks), mutant


# ------------------------------------------------------------------------------------------------ cast_colsum model and mutants
def cast_colsum_model(dy, p, seed, site, sms=132, mutant=None):
    """fp32 model of cast_colsum_f32_bf16_kernel on its cast_colsum_grid: per-chunk sums of the bf16 output, then the chunks in order"""
    T, D = dy.shape
    cy = min(-(-8 * sms // -(-D // 128)), -(-T // 32))
    rows_per = -(-T // cy)
    drop = torch.from_numpy(dr.drop_mask(np.arange(T), D, p, seed, site))
    sc = float(np.float32(dr.keep_scale(p)[1]))
    dyb = torch.where(drop, torch.zeros(()), dy * sc).bfloat16()
    out = torch.full((T, D), float("nan")).bfloat16()
    summed = dy.bfloat16() if mutant == "db_undropped" else dyb
    total = torch.zeros(D)
    for r0 in range(0, T, rows_per):
        r1 = min(T, r0 + rows_per)
        rows = []
        for ty in range(8):
            r = r0 + ty
            while r + 24 < r1:
                rows += [r, r + 8, r + 16, r + 24]
                r += 32
            if mutant != "skip_chunk_tail":
                rows += list(range(r, r1, 8))
        rows = torch.tensor(sorted(rows), dtype=torch.long)
        out[rows] = dyb[rows]
        total += summed[rows].float().sum(0)
    return out, total


@pytest.mark.parametrize("mutant", [None, "db_undropped", "skip_chunk_tail"])
def test_cast_colsum_model_and_mutants(mutant):
    """T = 50 rows in two chunks of 25: most rows of a chunk are in its tail loop"""
    g = torch.Generator().manual_seed(6)
    T, D, seed, site = 50, 64, 7, 10
    dy = torch.randint(-64, 65, (T, D), generator=g).float() / 64
    oks = []
    for p in (0.0, 0.5):
        out, db = cast_colsum_model(dy, p, seed, site, mutant=mutant)
        ref = hr.cast_colsum(dy, p, seed, site)
        oks.append(torch.equal(out, ref["dyb_exact"]) and torch.equal(db.double(), ref["db"]) and _ok([(db, ref["db"], ref["a_db"])]))
    assert all(oks) == (mutant is None), (mutant, oks)


# ------------------------------------------------------------------------------------------------ attention model and mutants
def attn_model(P, w, pad, H, zp, dO, mutant=None):
    """fp32 model of the HSTU attention kernels: 64-key tiles, A and dS packed to bf16 before their MMAs, fp32 accumulation"""
    B, L, D4 = P.shape
    D = D4 // 4
    hs = lambda t: t.float().reshape(B, L, H, D // H).transpose(1, 2)      # noqa: E731
    _, V, Q, K = P.split(D, -1)
    q, k, v, do = hs(Q), hs(K), hs(V), hs(dO)
    ii = torch.arange(L)
    i, j = ii[:, None], ii[None, :]
    causal = (j <= i) | ((j == i + 1) if mutant == "key_i_plus_1" else False)
    if mutant == "diag_dropped":
        causal = causal & (j != i)
    keyok = torch.ones(B, L, dtype=torch.bool) if mutant == "padded_key" else ~pad
    valid = causal[None, None] & keyok[:, None, None, :]
    if mutant == "last_partial_block" and L % 8:
        valid = valid & (j < L // 8 * 8)[None, None]
    x = q @ k.transpose(-1, -2) + w
    A = torch.where(valid, x * torch.sigmoid(x), torch.zeros(()))
    dS = torch.where(valid, (do @ v.transpose(-1, -2)) * hr.dsilu(x), torch.zeros(()))
    Ab, dSb = A.bfloat16().float(), dS.bfloat16().float()
    O = torch.zeros_like(q)
    dq = torch.zeros_like(q)
    for t0 in range(0, L, 64):
        O += Ab[..., t0:t0 + 64] @ v[:, :, t0:t0 + 64]
        dq += dSb[..., t0:t0 + 64] @ k[:, :, t0:t0 + 64]
    dk = (Ab if mutant == "dK_from_A" else dSb).transpose(-1, -2) @ q
    dv = Ab.transpose(-1, -2) @ do
    _, zV, zQ, zK = zp.split(D, -1)
    mg = lambda t: t.transpose(1, 2).reshape(B, L, D)                      # noqa: E731
    out = {"O": mg(O).bfloat16(), "dV": (mg(dv) * hr.dsilu(zV.float())).bfloat16(), "dK": (mg(dk) * hr.dsilu(zK.float())).bfloat16()}
    out["dQ"] = (mg(dq) * (1 if mutant == "dQ_no_dsilu" else hr.dsilu(zQ.float()))).bfloat16()
    return out


ATTN_MUTANTS = ["diag_dropped", "key_i_plus_1", "padded_key", "last_partial_block", "dQ_no_dsilu", "dK_from_A"]


@pytest.mark.parametrize("mutant", [None] + ATTN_MUTANTS)
def test_attention_model_and_mutants(mutant):
    """L = 65 (a second key tile holding one key, a partial 8-key block) and L = 130, at d/H = 32 and 64"""
    oks = []
    for B, L, D, H in ((3, 65, 64, 2), (3, 130, 128, 2)):
        zp, P, dO, pad, w = _attn_inputs(B, L, D, H, seed=L)
        got = attn_model(P, w, pad, H, zp, dO, mutant)
        ref = hr.attention(P, w, hr.causal_valid(pad), H, zp, dO)
        oks.append(_ok([(got[n], ref[n], ref["a_" + n]) for n in ("O", "dV", "dQ", "dK")]))
    assert all(oks) == (mutant is None), (mutant, oks)


# ------------------------------------------------------------------------------------------------ Adam model and mutants
def adam_model(p0, g0, m0, v0, t, lr, b1, b2, eps, wd, gs, mutant=None):
    """numpy fp32 model of adam_tick_kernel + adam_step_kernel -> p, m, v, bc1, bc2 and the bf16 mirror"""
    f = np.float32
    p0, g0, m0, v0 = (a.numpy().astype(f) for a in (p0, g0, m0, v0))
    lr, b1, b2, eps, wd, gs = (f(a) for a in (lr, b1, b2, eps, wd, gs))
    g = g0 if mutant == "no_grad_scale" else g0 * gs
    if wd != 0 and mutant != "adamw":
        g = g + wd * p0
    m = b1 * m0 + (f(1) - b1) * g
    v = b2 * v0 + (f(1) - b2) * g * g
    tt = f(t - 1 if mutant == "bc_behind" else t)
    bc1, bc2 = f(1) - np.power(b1, tt), f(1) - np.power(b2, tt)
    with np.errstate(divide="ignore", invalid="ignore"):
        ss = lr / bc1
        den = np.sqrt(v / bc2 + eps) if mutant == "eps_in_sqrt" else np.sqrt(v) * (f(1) / np.sqrt(bc2)) + eps
        p = p0 - ss * (m / den)
    if mutant == "adamw":
        p = p - lr * wd * p0
    pt = torch.from_numpy(p.astype(f))
    mirror = (pt.view(torch.int32) & -65536).view(torch.float32).bfloat16() if mutant == "mirror_trunc" else pt.bfloat16()
    return dict(p=pt, m=torch.from_numpy(m), v=torch.from_numpy(v), bc1=torch.tensor([bc1]), bc2=torch.tensor([bc2]), mirror=mirror)


ADAM_MUTANTS = ["bc_behind", "eps_in_sqrt", "adamw", "no_grad_scale", "mirror_trunc"]


@pytest.mark.parametrize("mutant", [None] + ADAM_MUTANTS)
def test_adam_model_and_mutants(mutant):
    g = torch.Generator().manual_seed(8)
    n = 4096
    p0 = torch.randn(n, generator=g)
    g0 = torch.randn(n, generator=g) * 10.0 ** -torch.randint(0, 6, (n,), generator=g).float()
    m0, v0 = 1e-3 * torch.randn(n, generator=g), 1e-6 * torch.rand(n, generator=g)
    oks = []
    for t, wd, gs in ((1, 0.0, 1.0), (2, 1e-2, 0.125), (10, 1e-2, 0.125), (1000, 0.0, 0.125)):
        got = adam_model(p0, g0, m0, v0, t, 1e-3, 0.9, 0.999, 1e-8, wd, gs, mutant)
        ref = hr.adam(p0, g0, m0, v0, t, 1e-3, 0.9, 0.999, 1e-8, wd, gs)
        ok = _ok([(got[k], ref[k], ref["a_" + k]) for k in ("p", "m", "v")] +
                 [(got[k], torch.tensor([ref[k]]), torch.tensor([ref["a_" + k]])) for k in ("bc1", "bc2")])
        oks.append(ok and torch.equal(got["mirror"], got["p"].bfloat16()))
    assert all(oks) == (mutant is None), (mutant, oks)


def test_layouts_restate_the_carve_order():
    """256-byte aligned regions in carve order; the saved blob's size at the benchmark's block shape"""
    sl, wl = hr.saved_layout(25600, 128), hr.work_layout(25600, 128)
    assert [k for k in sl if k != "bytes"] == ["xb", "zp", "P", "O", "st1", "x1", "xn", "st2", "z1", "hact"]
    assert all(v[0] % 256 == 0 for k, v in sl.items() if k != "bytes")
    T, D = 25600, 128
    assert sl["bytes"] == T * D * (2 + 8 + 8 + 2 + 4 + 2 + 8 + 8) + 2 * T * 2 * 4
    assert wl["dzp"][0] == T * D * (2 + 8 + 4 + 4 + 2) and wl["bytes"] == T * D * (2 + 8 + 4 + 4 + 2 + 8)
    assert math.prod(wl["dzp"][2]) == T * 4 * D
