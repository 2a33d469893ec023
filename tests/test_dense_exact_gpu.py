"""The linear GEMM epilogues, the weight-gradient GEMM and bias sums, LayerNorm, RMS norm and the embedding gather / scatter
against the fp64 references of tests/dense_reference.py, at their tile, tail, grid-wrap and piece edges; the embedding backward
against the numpy restatements of its fixed summation orders; and the SASRec training step's reproducibility.

Two kinds of operand: small integers times powers of two, with which every product, partial sum and fp32 output is exact, so
the kernel must equal the fp64 value bit for bit (a bf16 output its round-to-nearest-even) whatever its summation order; and
Gaussian operands, whose error must stay within the derived allowance.  `pytest -s` prints each case's worst ratio of error to
allowance."""
import math

import pytest
import torch

from tests import dense_reference as dr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _ints(shape, lo, hi, unit, g):
    """small integers in [lo, hi] times the power of two `unit` (fp32)"""
    return torch.randint(lo, hi + 1, shape, generator=g).float() * unit


def _report(tag, err):
    print(f"{tag}: {dr.fmt(err)}")


def _check(tag, err):
    _report(tag, err)
    assert not dr.violations(err), dr.fmt(err)


# ------------------------------------------------------------------------------------------------ linear
# N and K from {8, 24, 40, 72, 136, 200, 264} (tails of the 64-wide K box, of the 32-column epilogue chunks and of the 128-wide
# tiles) and {64, 512}; M cycles through {1, 127, 128, 129, 25600}.
LIN_NK = [(8, 264), (24, 200), (40, 136), (72, 72), (136, 40), (200, 24), (264, 8), (64, 512), (512, 64), (8, 8), (264, 264),
          (40, 512), (512, 40), (72, 200), (200, 72)]
LIN_M = [1, 127, 128, 129, 25600]
LIN_SHAPES = [(LIN_M[n % 5], N, K) for n, (N, K) in enumerate(LIN_NK)]


def _lin_operands(M, N, K, exact, seed):
    """exact: x in [-4, 4] / 8, w in [-3, 3] / 4, bias in [-64, 64] / 32 - every |acc| < 2^9 on a 2^-5 grid, so fp32 holds every
    partial sum and z + bias exactly.  Otherwise x ~ N(0, 1), w ~ 0.1 N(0, 1), bias ~ N(0, 1)."""
    g = torch.Generator().manual_seed(seed)
    if exact:
        x, w, b = _ints((M, K), -4, 4, 0.125, g), _ints((N, K), -3, 3, 0.25, g), _ints((N,), -64, 64, 1 / 32, g)
    else:
        x, w, b = torch.randn(M, K, generator=g), 0.1 * torch.randn(N, K, generator=g), torch.randn(N, generator=g)
    return x.bfloat16().to(DEV), w.bfloat16().to(DEV), b.to(DEV)


@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("M,N,K", LIN_SHAPES)
def test_linear_forward_vs_fp64(M, N, K, exact):
    """z = bf16(x w^T + bias) and a = bf16(dropout(ACT(z))) for ACT none / SiLU / ReLU.  Exact operands (p in {0, 0.5}): z and the
    ReLU output equal the RNE of the exact value.  Gaussian operands (p in {0, 0.2}): within the allowance; the ReLU output still
    equals its restatement from the kernel's own z."""
    import genrec_b200.functional as Fn
    n = LIN_SHAPES.index((M, N, K))
    p = (0.0, 0.5)[n % 2] if exact else (0.0, 0.2)[n % 2]
    seed, site = 77 + n, 5
    x, w, b = _lin_operands(M, N, K, exact, 1000 * n + exact)
    for act in (0, 1, 2):
        z, a = Fn.linear_fwd(x, w, b, act, p=p, seed=seed, site=site)
        ref = dr.linear_forward(x, w, b, act, z, p, seed, site)
        if exact:
            assert torch.equal(z, dr.rne_bf16(ref["z"])), f"z act={act}"
        err = {"z": dr.worst(z, ref["z"], ref["a_z"])}
        if act:
            err["a"] = dr.worst(a, ref["a"], ref["a_a"])
            assert not bool(a[ref["a"] == 0].any())
        if act == 2:
            assert torch.equal(a, ref["a_exact"]), "relu output"
        _check(f"linear fwd M={M} N={N} K={K} act={act} p={p} exact={exact}", err)


@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("M,N,K", LIN_SHAPES[::2])
def test_linear_residual_vs_fp64(M, N, K, exact):
    """y = (res + dropout(x w^T + bias)) * row_scale in fp32, with and without row_scale (0, 1 and 1/2 per row)."""
    import genrec_b200.functional as Fn
    n = LIN_SHAPES.index((M, N, K))
    p = (0.0, 0.5)[n % 2] if exact else (0.0, 0.2)[n % 2]
    x, w, b = _lin_operands(M, N, K, exact, 2000 * n + exact)
    g = torch.Generator().manual_seed(n)
    res = (_ints((M, N), -512, 512, 1 / 64, g) if exact else torch.randn(M, N, generator=g)).to(DEV)
    rs = (torch.randint(0, 3, (M,), generator=g).float() / 2).to(DEV)
    for row_scale in (None, rs):
        y = Fn.linear_residual_fwd(x, w, b, res, row_scale, p=p, seed=9 + n, site=6)
        ref = dr.linear_residual(x, w, b, res, row_scale, p, 9 + n, 6)
        if exact:
            assert torch.equal(y.double(), ref["y"]), f"row_scale={row_scale is not None}"
        _check(f"linear residual M={M} N={N} K={K} row_scale={row_scale is not None} p={p} exact={exact}",
               {"y": dr.worst(y, ref["y"], ref["a_y"])})


def tn_splits(T, N, K, sms):
    """the k-splits tn_plan (csrc/tc_tn_group.cuh) gives dW [N, K] += dy^T x over T tokens, launched alone"""
    kb = (T + 63) // 64
    tiles = ((N + 127) // 128) * ((K + 127) // 128)
    splits = max(1, (int(2.0 * sms + 0.5) + tiles - 1) // tiles)
    splits = min(splits, max(1, kb // 4))
    per = (kb + splits - 1) // splits
    return (kb + per - 1) // per


# dW through one k-split (T <= 511) and through many (T = 25600), with K % 32 != 0 on both sides (the scalar tail of the
# one-split store); dx with and without the residual
LIN_BWD = [(1, 8, 264), (127, 40, 136), (129, 264, 40), (129, 72, 200), (511, 512, 24), (25600, 8, 264), (25600, 64, 64),
           (25600, 512, 512), (25600, 200, 40), (25600, 136, 72), (128, 24, 8)]


@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("T,N,K", LIN_BWD)
def test_linear_backward_vs_fp64(T, N, K, exact):
    """dx = dy W (+ res), dW = dy^T x, db = colsum(dy) into zeroed outputs.  Exact operands: bit for bit (|dW| < 2^15 on a 2^-6
    grid over 25,600 tokens, so a lost k-split or tail column cannot hide); Gaussian: within the fp32 accumulation allowance."""
    import genrec_b200.functional as Fn
    n = LIN_BWD.index((T, N, K))
    g = torch.Generator().manual_seed(3000 + n)
    if exact:
        dy, x = _ints((T, N), -3, 3, 0.25, g), _ints((T, K), -4, 4, 0.125, g)
        w, res = _ints((N, K), -3, 3, 0.25, g), _ints((T, K), -256, 256, 1 / 32, g)
    else:
        dy, x, w, res = 0.1 * torch.randn(T, N, generator=g), torch.randn(T, K, generator=g), 0.1 * torch.randn(N, K, generator=g), \
            torch.randn(T, K, generator=g)
    dy, x, w, res = dy.bfloat16().to(DEV), x.bfloat16().to(DEV), w.bfloat16().to(DEV), res.to(DEV)
    for r in (None, res):
        dx, dw, db = Fn.linear_bwd(dy, w, x, dx_residual=r)
        ref = dr.linear_backward(dy, w, x, r)
        got = {"dx": dx, "dw": dw, "db": db}
        if exact:
            for k in got:
                assert torch.equal(got[k].double(), ref[k]), k
        _check(f"linear bwd T={T} N={N} K={K} splits={tn_splits(T, N, K, _sms())} res={r is not None} exact={exact}",
               dr.errors(got, ref, ("dx", "dw", "db")))


def test_linear_backward_cases_reach_both_dw_paths():
    sms = _sms()
    splits = [tn_splits(T, N, K, sms) for T, N, K in LIN_BWD]
    assert any(s == 1 and K % 32 for s, (_, _, K) in zip(splits, LIN_BWD))
    assert any(s > 1 and K % 32 for s, (_, _, K) in zip(splits, LIN_BWD))
    assert any(s > 8 for s in splits)


# ------------------------------------------------------------------------------------------------ LayerNorm / RMS norm
def _norm_T():
    """T in {1, 7, 8, 9} and just below, at and above the row counts where the backward grid (3 x SMs CTAs of 8 rows) and the
    forward grid (8 x SMs CTAs of 8 rows) start to wrap"""
    s = _sms()
    return [1, 7, 8, 9] + [8 * k * s + d for k in (3, 8) for d in (-1, 0, 1)]


def _norm_inputs(T, D, seed):
    """x ~ N(0, 1) with every third row offset by 1000 (|mean| >> std: a one-pass variance loses it), g ~ 1 + 0.2 N, b ~ 0.2 N"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, D, generator=g)
    x[::3] += 1000 * torch.sign(torch.randn(x[::3].shape[0], 1, generator=g))
    gam, bet = 1 + 0.2 * torch.randn(D, generator=g), 0.2 * torch.randn(D, generator=g)
    dy, res = torch.randn(T, D, generator=g), torch.randn(T, D, generator=g)
    return [t.to(DEV) for t in (x, gam, bet, dy, res)]


@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("Ti", range(10))
def test_layernorm_vs_fp64(D, Ti):
    import genrec_b200.functional as Fn
    T = _norm_T()[Ti]
    x, gam, bet, dy, res = _norm_inputs(T, D, T + D)
    yb, yf, st = Fn.layernorm_fwd(x, gam, bet, 1e-8, want_bf16=True, want_f32=True)
    ref = dr.layernorm_forward(x, gam, bet, 1e-8)
    err = {"y bf16": dr.worst(yb, ref["y"], ref["a_y16"]), "y fp32": dr.worst(yf, ref["y"], ref["a_y32"]),
           "mean": dr.worst(st[:, 0], ref["mean"], ref["a_mean"]), "rstd": dr.worst(st[:, 1], ref["rstd"], ref["a_rstd"])}
    r = res if Ti % 2 else None
    dx, dg, db = Fn.layernorm_bwd(dy, x, st, gam, r)
    err.update(dr.errors({"dx": dx, "dg": dg, "db": db}, dr.layernorm_backward(dy, x, st, gam, r), ("dx", "dg", "db")))
    _check(f"layernorm T={T} D={D} res={r is not None}", err)


@pytest.mark.parametrize("D", [64, 128, 256, 384])
@pytest.mark.parametrize("Ti", range(10))
def test_rmsnorm_vs_fp64(D, Ti):
    import genrec_b200.functional as Fn
    T = _norm_T()[Ti]
    x, w, _, dy, res = _norm_inputs(T, D, 7 * T + D)
    yb, yf, rstd = Fn.rmsnorm_fwd(x, w, 1e-6, want_bf16=True, want_f32=True)
    ref = dr.rmsnorm_forward(x, w, 1e-6)
    err = {"y bf16": dr.worst(yb, ref["y"], ref["a_y16"]), "y fp32": dr.worst(yf, ref["y"], ref["a_y32"]),
           "rstd": dr.worst(rstd, ref["rstd"], ref["a_rstd"])}
    r = res if Ti % 2 == 0 else None
    dx, dw = Fn.rmsnorm_bwd(dy, x, rstd, w, r)
    err.update(dr.errors({"dx": dx, "dw": dw}, dr.rmsnorm_backward(dy, x, rstd, w, r), ("dx", "dw")))
    _check(f"rmsnorm T={T} D={D} res={r is not None}", err)


@pytest.mark.parametrize("D", [32, 96, 192, 384, 512])
def test_layernorm_rejects_unsupported_width(D):
    import genrec_b200.functional as Fn
    from genrec_b200._lib import GrbError
    x, gam, _, dy, _ = _norm_inputs(16, D, D)
    with pytest.raises(GrbError):
        Fn.layernorm_fwd(x, gam, gam, 1e-8)
    st = torch.zeros(16, 2, device=DEV)
    with pytest.raises(GrbError):
        Fn.layernorm_bwd(dy, x, st, gam)


@pytest.mark.parametrize("D", [32, 96, 192, 320, 512])
def test_rmsnorm_rejects_unsupported_width(D):
    import genrec_b200.functional as Fn
    from genrec_b200._lib import GrbError
    x, w, _, dy, _ = _norm_inputs(16, D, D)
    with pytest.raises(GrbError):
        Fn.rmsnorm_fwd(x, w, 1e-6)
    with pytest.raises(GrbError):
        Fn.rmsnorm_bwd(dy, x, torch.ones(16, device=DEV), w)


# ------------------------------------------------------------------------------------------------ embedding
def _embed_ids(B, L, big_run, seed):
    """[B, L] ids, shuffled: id 0 fills the first sorted piece (32 positions, fewer for tiny T) and id 1 the next two, so both runs
    end exactly on a piece boundary; id 2 fills `big_run` positions (more than 32 pieces cross embed_bwd_run_kernel's ballot
    window); the rest are drawn from about T / 4 ids, so runs of several tokens straddle piece boundaries."""
    T = B * L
    g = torch.Generator().manual_seed(seed)
    n0 = min(32, T // 4)
    n1 = 64 if T >= 256 else 0
    head = [0] * n0 + [1] * n1 + [2] * big_run
    V = max(8, T // 4)
    rest = torch.randint(3, V, (T - len(head),), generator=g)
    ids = torch.cat([torch.tensor(head, dtype=torch.int64), rest])[torch.randperm(T, generator=g)]
    return ids.view(B, L), V


def _big_T_shape():
    """B x L with B L > 8 x 8 x SMs x 32: more 32-token pieces than the piece kernel's grid has warps"""
    L = 50
    return 64 * 32 * _sms() // L + 2, L


# (D, (B, L), scale sqrt(D), p, position table, mask_pad_rows); T in {31, 32, 33, 1024, 1025} and 2400 (a 1,100-token run)
EMB_SHAPES = [(1, 31), (2, 16), (3, 11), (32, 32), (25, 41), (48, 50)]
EMB_CASES = [(D, EMB_SHAPES[(n + k) % 6], n % 2 == 1, (0.0, 0.2, 0.5)[(n + k) % 3], (n + k) % 4 != 3, k % 2)
             for k, D in enumerate((4, 36, 64, 132, 256)) for n in range(6)]


def _embed_run(ids, E, pos, L, scale, mask, p, seed, dE0, dpos0, dx):
    """forward through EmbedFn, backward into the sinks dE0 / dpos0 (cloned) -> (x, pad, dE, dpos)"""
    import genrec_b200.functional as Fn
    dE, dpos = dE0.clone(), (dpos0.clone() if dpos0 is not None else None)
    table = E.clone().requires_grad_(True)
    x, pad = Fn.EmbedFn.apply(ids, table, pos, scale, mask, p, seed, None, (dE, dpos))
    x.backward(dx.view_as(x))
    return x.detach(), pad, dE, dpos


def _embed_case(D, B, L, scale, p, with_pos, mask, big_run, seed):
    T = B * L
    ids, V = _embed_ids(B, L, big_run, seed)
    g = torch.Generator().manual_seed(seed + 1)
    E, dx = torch.randn(V, D, generator=g), torch.randn(T, D, generator=g)
    P = L + 3
    pos = torch.randn(P, D, generator=g).to(DEV) if with_pos else None
    dE0 = torch.randn(V, D, generator=g)
    dpos0 = torch.randn(P, D, generator=g).to(DEV) if with_pos else None
    args = (ids.to(DEV), E.to(DEV), pos, L, scale, mask, p, 4321 + seed, dE0.to(DEV), dpos0, dx.to(DEV))
    first, second = _embed_run(*args), _embed_run(*args)
    for name, a, b in zip(("x", "pad", "dE", "dpos"), first, second):
        assert a is None or torch.equal(a, b), f"{name} differs between two runs"
    x, pad, dE, dpos = first
    fwd = dr.embed_forward(ids, E, pos, L, scale, mask, p, 4321 + seed)
    bwd = dr.embed_backward(ids, dx, L, V, P if with_pos else 0, scale, mask, p, 4321 + seed, dE0, dpos0)
    assert torch.equal(pad.view(-1).cpu().bool(), fwd["pad"])
    assert torch.equal(dE[0].cpu(), dE0[0]), "row 0 of dE changed"
    err = {"x": dr.worst(x.view(T, D), fwd["x"], fwd["a_x"]), "dE": dr.worst(dE, bwd["dE"], bwd["a_dE"])}
    if with_pos:
        err["dpos"] = dr.worst(dpos, bwd["dpos"], bwd["a_dpos"])
    if scale == 1.0 and p in (0.0, 0.5):
        # E + pos rounds once in fp32 (a fused E * 1 + pos alike), the keep scale 2 and the pad mask are exact
        e = E[ids.view(-1)] + (pos.cpu()[torch.arange(T) % L] if with_pos else 0)
        live = (ids.view(-1, 1) != 0).float() if mask else 1.0
        assert torch.equal(x.view(T, D).cpu(), e * dr.keep(range(T), D, p, 4321 + seed, dr.SITE_EMBED).float() * live), "x"
    if scale == 1.0 and p == 0.0:
        assert torch.equal(dE.cpu(), dr.embed_dE_fixed_order(ids, dx, dE0)), "dE is not the fixed-order sum"
        if with_pos:
            assert torch.equal(dpos.cpu(), dr.embed_dpos_fixed_order(ids, dx, L, mask, dpos0)), "dpos is not the ascending-b sum"
    _check(f"embed T={T} D={D} scale={scale:.3g} p={p} pos={with_pos} mask={mask} run={big_run}", err)


@pytest.mark.parametrize("D,BL,sqrt_scale,p,with_pos,mask", EMB_CASES)
def test_embedding_vs_fp64(D, BL, sqrt_scale, p, with_pos, mask):
    B, L = BL
    big = 1100 if B * L == 2400 else 0
    _embed_case(D, B, L, math.sqrt(D) if sqrt_scale else 1.0, p, with_pos, mask, big, D * 100 + B)


@pytest.mark.parametrize("D,mask", [(4, 1), (36, 0), (256, 1)])
def test_embedding_fixed_orders_at_hstu_setting(D, mask):
    """scale 1, p = 0 (HSTU's embedding), with and without a position table: dE and dpos equal the numpy fixed-order sums bit for
    bit, including one id filling 1,100 consecutive sorted positions."""
    for with_pos in (True, False):
        _embed_case(D, 48, 50, 1.0, 0.0, with_pos, mask, 1100, 17 + D)


def test_embedding_wraps_the_piece_grid():
    """More 32-token pieces than embed_bwd_piece_kernel has warps (and more tokens than the run kernel's grid has warps), with a
    run of 2,500 tokens; D = 4 keeps the restatement cheap."""
    B, L = _big_T_shape()
    assert B * L > 8 * 8 * _sms() * 32
    _embed_case(4, B, L, 1.0, 0.0, True, 1, 2500, 5)


def test_embedding_backward_rejects_wide_rows():
    import genrec_b200.functional as Fn
    from genrec_b200._lib import GrbError
    B, L, D = 2, 8, 260
    ids = torch.randint(1, 10, (B, L), device=DEV)
    table = torch.randn(10, D, device=DEV, requires_grad=True)
    x, _ = Fn.EmbedFn.apply(ids, table, None, 1.0, 1, 0.0, 0, None)
    ref = dr.embed_forward(ids, table.detach(), None, L, 1.0, 1)
    assert torch.equal(x.detach().view(B * L, D).cpu().double(), ref["x"])
    with pytest.raises(GrbError):
        x.backward(torch.ones_like(x))


# ------------------------------------------------------------------------------------------------ SASRec training step
def test_sasrec_training_step_is_reproducible():
    """Forward and backward of SASRec at configs[0] geometry (B = 128, L = 50, d = 64, 2 blocks, dropout 0.2), run twice from the
    same seeds: every .grad is the same bits, position_embedding.weight included."""
    from genrec_b200.sasrec import SASRec
    B, L, V = 128, 50, 1000
    torch.manual_seed(0)
    m = SASRec(V, L, 64, 2, 2, 256, dropout=0.2).to(DEV).train()
    g = torch.Generator().manual_seed(6)
    ids = torch.randint(1, V + 1, (B, L), generator=g)
    ids[torch.arange(L)[None, :] < torch.randint(0, L - 1, (B, 1), generator=g)] = 0      # left padding
    tg = torch.roll(ids, -1, 1)
    ids, tg = ids.to(DEV), tg.to(DEV)

    def run():
        torch.manual_seed(123)
        m._seed_dev = None
        m.zero_grad(set_to_none=True)
        m(ids, tg)[1].backward()
        return {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}

    first, second = run(), run()
    assert "position_embedding.weight" in first and len(first) > 20
    bad = [n for n in first if not torch.equal(first[n], second[n])]
    assert not bad, bad
