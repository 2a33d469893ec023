"""The references and checks of tests/dense_reference.py, without a GPU: each reference agrees with torch autograd in fp64, an fp32
model of each kernel passes its check, and a model with one planted defect - a mutant of what the check guards - fails it."""
import numpy as np
import pytest
import torch

from tests import dense_reference as dr

def _ints(shape, lo, hi, unit, g):
    return torch.randint(lo, hi + 1, shape, generator=g).float() * unit


# ------------------------------------------------------------------------------------------------ references vs autograd
def test_linear_reference_matches_autograd():
    g = torch.Generator().manual_seed(0)
    T, N, K = 37, 24, 40
    x, w, b = torch.randn(T, K, generator=g).bfloat16(), torch.randn(N, K, generator=g).bfloat16(), torch.randn(N, generator=g)
    dy, res = torch.randn(T, N, generator=g).bfloat16(), torch.randn(T, K, generator=g)
    xr, wr, br = (t.double().requires_grad_(True) for t in (x, w, b))
    z = xr @ wr.T + br
    z.backward(dy.double())
    ref = dr.linear_forward(x, w, b)
    assert torch.allclose(ref["z"], z.detach(), rtol=1e-12, atol=1e-12)
    bw = dr.linear_backward(dy, w, x, res)
    assert torch.allclose(bw["dx"], xr.grad + res.double(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(bw["dw"], wr.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(bw["db"], br.grad, rtol=1e-12, atol=1e-12)
    rs, res_n = torch.rand(T, generator=g), torch.randn(T, N, generator=g)
    y = dr.linear_residual(x, w, b, res_n, rs)["y"]
    assert torch.allclose(y, (res_n.double() + z.detach()) * rs.double()[:, None], rtol=1e-12, atol=1e-12)


def test_layernorm_reference_matches_autograd():
    g = torch.Generator().manual_seed(1)
    T, D = 20, 64
    x, gam, bet, dy = torch.randn(T, D, generator=g) + 5, torch.randn(D, generator=g), torch.randn(D, generator=g), torch.randn(T, D, generator=g)
    xr, gr, br = (t.double().requires_grad_(True) for t in (x, gam, bet))
    y = torch.nn.functional.layer_norm(xr, (D,), gr, br, 1e-8)
    y.backward(dy.double())
    f = dr.layernorm_forward(x, gam, bet, 1e-8)
    assert torch.allclose(f["y"], y.detach(), rtol=1e-10, atol=1e-10)
    st = torch.stack([f["mean"], f["rstd"]], 1)
    b = dr.layernorm_backward(dy, x, st, gam)
    for k, ref in (("dx", xr.grad), ("dg", gr.grad), ("db", br.grad)):
        assert torch.allclose(b[k], ref, rtol=1e-9, atol=1e-9), k


def test_rmsnorm_reference_matches_autograd():
    g = torch.Generator().manual_seed(2)
    T, D = 20, 384
    x, w, dy = torch.randn(T, D, generator=g), torch.randn(D, generator=g), torch.randn(T, D, generator=g)
    xr, wr = x.double().requires_grad_(True), w.double().requires_grad_(True)
    y = wr * (xr * torch.rsqrt((xr * xr).mean(1, keepdim=True) + 1e-6))
    y.backward(dy.double())
    f = dr.rmsnorm_forward(x, w, 1e-6)
    assert torch.allclose(f["y"], y.detach(), rtol=1e-12, atol=1e-12)
    b = dr.rmsnorm_backward(dy, x, f["rstd"], w)
    assert torch.allclose(b["dx"], xr.grad, rtol=1e-9, atol=1e-9)
    assert torch.allclose(b["dw"], wr.grad, rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("mask,p", [(0, 0.0), (1, 0.5)])
def test_embedding_reference_matches_autograd(mask, p):
    g = torch.Generator().manual_seed(3)
    B, L, V, D, scale, seed = 3, 7, 9, 8, 2.0 ** 1.5, 11
    ids = torch.randint(0, V, (B, L), generator=g)
    E, pos, dx = torch.randn(V, D, generator=g), torch.randn(L + 2, D, generator=g), torch.randn(B * L, D, generator=g)
    Er, pr = E.double().requires_grad_(True), pos.double().requires_grad_(True)
    km = dr.keep(range(B * L), D, p, seed, dr.SITE_EMBED)
    live = (~((ids.view(-1) == 0) & bool(mask))).double()[:, None]
    x = (torch.nn.functional.embedding(ids.view(-1), Er) * float(np.float32(scale)) + pr[torch.arange(B * L) % L]) * km * live
    x.backward(dx.double())
    f = dr.embed_forward(ids, E, pos, L, scale, mask, p, seed)
    assert torch.allclose(f["x"], x.detach(), rtol=1e-12, atol=1e-12)
    b = dr.embed_backward(ids, dx, L, V, L + 2, scale, mask, p, seed)
    gE = Er.grad.clone()
    gE[0] = 0                                                 # the table's padding row takes no gradient
    assert torch.allclose(b["dE"], gE, rtol=1e-12, atol=1e-12)
    assert torch.allclose(b["dpos"], pr.grad, rtol=1e-12, atol=1e-12)


# ------------------------------------------------------------------------------------------------ fp32 models and their mutants
def _lin_model(x, w, b, act, p, seed, site, mutant=None):
    """fp32 model of TcEpiBiasAct: (z bf16, a bf16)"""
    K, N = x.shape[1], w.shape[0]
    xs, ws = x.float(), w.float()
    if mutant == "k_tail":                                   # the partial last 64-wide K box never loaded
        kk = K // 64 * 64
        xs, ws = xs[:, :kk], ws[:, :kk]
    acc = xs @ ws.T
    bb = b.clone()
    if mutant == "bias_last_chunk":                          # the last 32-column epilogue chunk without its bias
        bb[(N - 1) // 32 * 32:] = 0
    z32 = acc + bb
    z = z32.bfloat16()
    zin = z32 if mutant == "z_unrounded" else z.float()
    f = torch.relu(zin) if act == 2 else zin * torch.sigmoid(zin)
    km = dr.keep(range(x.shape[0]), N, p, seed, site).float()
    return z, (f * km).bfloat16()


@pytest.mark.parametrize("mutant", [None, "k_tail", "bias_last_chunk", "z_unrounded"])
def test_linear_forward_model_and_mutants(mutant):
    """exact operands at K = 136 (a 64-wide K box tail of 8) and N = 40 (a last chunk of 8 columns): the model equals the RNE of the
    exact value; each mutant breaks an exact check or the allowance.  z_unrounded shows at p = 0.2, whose keep scale is not a power
    of two (ReLU commutes with the rounding otherwise), and in SiLU."""
    g = torch.Generator().manual_seed(4)
    T, N, K = 129, 40, 136
    x, w, b = _ints((T, K), -4, 4, 0.125, g).bfloat16(), _ints((N, K), -3, 3, 0.25, g).bfloat16(), torch.randn(N, generator=g)
    if mutant != "z_unrounded":
        b = _ints((N,), -64, 64, 1 / 32, g)
    fails = []
    for act, p in ((2, 0.2), (1, 0.0)):
        z, a = _lin_model(x, w, b, act, p, 3, 5, mutant)
        ref = dr.linear_forward(x, w, b, act, z, p, 3, 5)
        ok_z = (torch.equal(z, dr.rne_bf16(ref["z"])) if mutant != "z_unrounded" else True) and dr.worst(z, ref["z"], ref["a_z"]) <= dr.TOL
        ok_a = dr.worst(a, ref["a"], ref["a_a"]) <= dr.TOL and (act != 2 or torch.equal(a, ref["a_exact"]))
        fails.append(not (ok_z and ok_a))
    assert any(fails) == (mutant is not None), (mutant, fails)


def _dw_model(dy, x, splits, mutant=None):
    """fp32 model of the weight-gradient GEMM: per-split sums, then the splits in order"""
    T = dy.shape[0]
    per = -(-T // splits)
    parts = [dy[s:s + per].float().T @ x[s:s + per].float() for s in range(0, T, per)]
    if mutant == "lost_split":
        parts = parts[:-2] + parts[-1:]
    out = torch.zeros_like(parts[0])
    for q in parts:
        out = out + q
    return out


@pytest.mark.parametrize("exact", [True, False])
@pytest.mark.parametrize("mutant", [None, "lost_split"])
def test_weight_gradient_model_and_lost_split(mutant, exact):
    """T = 25,600, 100 splits of 256 tokens: a lost split fails the exact check; the fp32 accumulation allowance alone does not see
    it with Gaussian operands (why the exact operands are there), so only the unmutated model is required to pass it."""
    g = torch.Generator().manual_seed(5)
    T, N, K = 25600, 16, 24
    if exact:
        dy, x = _ints((T, N), -3, 3, 0.25, g).bfloat16(), _ints((T, K), -4, 4, 0.125, g).bfloat16()
    else:
        dy, x = (0.1 * torch.randn(T, N, generator=g)).bfloat16(), torch.randn(T, K, generator=g).bfloat16()
    w = torch.zeros(N, K).bfloat16()
    dw = _dw_model(dy, x, 100, mutant)
    ref = dr.linear_backward(dy, w, x)
    if mutant is None:
        assert dr.worst(dw, ref["dw"], ref["a_dw"]) <= dr.TOL
        if exact:
            assert torch.equal(dw.double(), ref["dw"])
    elif exact:
        assert not torch.equal(dw.double(), ref["dw"])


def _ln_model(x, g, b, eps, mutant=None):
    """fp32 model of ln_fwd_kernel: (y fp32, stats [T, 2])"""
    mean = x.mean(1, keepdim=True)
    if mutant == "one_pass":
        var = (x * x).mean(1, keepdim=True) - mean * mean
    else:
        var = ((x - mean) ** 2).mean(1, keepdim=True)
    rstd = torch.rsqrt(var + eps)
    y = (x - mean) * rstd * g + b
    if mutant == "skip_last_row":                            # a warp's last grid-stride iteration never runs
        y[-1] = 0
    return y, torch.cat([mean, rstd], 1)


def _ln_bwd_model(dy, x, st, g, mutant=None):
    m, r = st[:, 0:1], st[:, 1:2]
    xh = (x - m) * r
    gg = dy * g
    dx = r * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True))
    keep_rows = slice(None) if mutant != "skip_last_row" else slice(0, -1)
    if mutant == "skip_last_row":
        dx[-1] = 0
    return dx, (dy[keep_rows] * xh[keep_rows]).sum(0), dy[keep_rows].sum(0)


def _ln_case(T, D, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, D, generator=g)
    x[::3] += 1000 * torch.sign(torch.randn(x[::3].shape[0], 1, generator=g))
    return x, 1 + 0.2 * torch.randn(D, generator=g), 0.2 * torch.randn(D, generator=g), torch.randn(T, D, generator=g)


@pytest.mark.parametrize("D", [64, 256])
@pytest.mark.parametrize("mutant", [None, "one_pass", "skip_last_row"])
def test_layernorm_model_and_mutants(mutant, D):
    T = 8 * 8 * 132 + 1
    x, gam, bet, dy = _ln_case(T, D, D)
    y, st = _ln_model(x, gam, bet, 1e-8, mutant)
    f = dr.layernorm_forward(x, gam, bet, 1e-8)
    err = {"y32": dr.worst(y, f["y"], f["a_y32"]), "y16": dr.worst(y.bfloat16(), f["y"], f["a_y16"]),
           "mean": dr.worst(st[:, 0], f["mean"], f["a_mean"]), "rstd": dr.worst(st[:, 1], f["rstd"], f["a_rstd"])}
    dx, dg, db = _ln_bwd_model(dy, x, st, gam, mutant)
    err.update(dr.errors({"dx": dx, "dg": dg, "db": db}, dr.layernorm_backward(dy, x, st, gam), ("dx", "dg", "db")))
    assert bool(dr.violations(err)) == (mutant is not None), (mutant, dr.fmt(err))


@pytest.mark.parametrize("D", [64, 384])
@pytest.mark.parametrize("mutant", [None, "skip_last_row"])
def test_rmsnorm_model_and_mutants(mutant, D):
    T = 8 * 3 * 132 + 1
    x, w, _, dy = _ln_case(T, D, D + 1)
    r = torch.rsqrt((x * x).mean(1, keepdim=True) + 1e-6)
    y = w * (x * r)
    xh = x * r
    gg = dy * w
    dx = r * (gg - xh * (gg * xh).mean(1, keepdim=True))
    if mutant == "skip_last_row":
        y[-1] = 0
        dx[-1] = 0
    f = dr.rmsnorm_forward(x, w, 1e-6)
    err = {"y32": dr.worst(y, f["y"], f["a_y32"]), "y16": dr.worst(y.bfloat16(), f["y"], f["a_y16"]),
           "rstd": dr.worst(r[:, 0], f["rstd"], f["a_rstd"])}
    err.update(dr.errors({"dx": dx, "dw": (dy * xh).sum(0)}, dr.rmsnorm_backward(dy, x, r[:, 0], w), ("dx", "dw")))
    assert bool(dr.violations(err)) == (mutant is not None), (mutant, dr.fmt(err))


def _embed_case(seed, T=2400, L=50, run=1100):
    g = torch.Generator().manual_seed(seed)
    V = T // 4
    ids = torch.cat([torch.zeros(32, dtype=torch.int64), torch.ones(64, dtype=torch.int64), torch.full((run,), 2),
                     torch.randint(3, V, (T - 96 - run,), generator=g)])[torch.randperm(T, generator=g)]
    return ids.view(-1, L), V, torch.randn(T, 36, generator=g), torch.randn(V, 36, generator=g), torch.randn(L + 3, 36, generator=g)


def _dE_lost_last_piece(ids, dx, dE0):
    """the fixed-order sum with the last piece of every run that spans more than one piece lost"""
    idf = ids.reshape(-1).numpy()
    g = dx.numpy()
    dE = dE0.numpy().copy()
    order = np.argsort(idf, kind="stable")
    sid = idf[order]
    starts = np.flatnonzero(np.r_[True, sid[1:] != sid[:-1]])
    for p0, p1 in zip(starts, np.r_[starts[1:], len(order)]):
        if sid[p0] == 0:
            continue
        last = (p1 - 1) // 32 * 32
        stop = last if last > p0 else p1
        dE[sid[p0]] += np.cumsum(g[order[p0:stop]], axis=0, dtype=np.float32)[-1]
    return torch.from_numpy(dE)


@pytest.mark.parametrize("mutant", [None, "lost_last_piece"])
def test_embedding_dE_order_and_lost_piece(mutant):
    ids, V, dx, dE0, _ = _embed_case(6)
    ref = dr.embed_backward(ids, dx, 50, V, 0, 1.0, 1, dE0=dE0)
    got = dr.embed_dE_fixed_order(ids, dx, dE0) if mutant is None else _dE_lost_last_piece(ids, dx, dE0)
    assert torch.equal(got[0], dE0[0])
    assert (dr.worst(got, ref["dE"], ref["a_dE"]) <= dr.TOL) == (mutant is None)


@pytest.mark.parametrize("shift", [0, -1, 1])
@pytest.mark.parametrize("mask", [0, 1])
def test_embedding_dpos_order_and_shifted_row(shift, mask):
    ids, V, dx, _, dpos0 = _embed_case(7)
    L = 50
    ref = dr.embed_backward(ids, dx, L, V, L + 3, 1.0, mask, dpos0=dpos0)
    got = dr.embed_dpos_fixed_order(ids, dx, L, mask, dpos0)
    if shift:
        got = dpos0.clone()
        live = ~((ids.reshape(-1) == 0) & bool(mask))
        rows = (torch.arange(dx.shape[0]) % L + shift) % L
        got.index_add_(0, rows[live], dx[live])
    assert (dr.worst(got, ref["dpos"], ref["a_dpos"]) <= dr.TOL) == (shift == 0)


def test_fixed_order_restatements_are_orders_not_values():
    """At a piece boundary the restatement's order matters: it differs from a plain left-to-right sum over all of a run's tokens
    for some id, so a kernel summing in any other order would not match it bit for bit."""
    ids, V, dx, dE0, _ = _embed_case(8)
    fixed = dr.embed_dE_fixed_order(ids, dx, torch.zeros_like(dE0))
    idf = ids.reshape(-1)
    order = torch.sort(idf, stable=True).indices
    plain = np.zeros((V, dx.shape[1]), dtype=np.float32)
    g = dx.numpy()
    for t in order.tolist():
        if idf[t] != 0:
            plain[idf[t]] += g[t]
    assert not torch.equal(fixed, torch.from_numpy(plain))
    assert torch.equal(fixed[0], torch.zeros(dx.shape[1]))
