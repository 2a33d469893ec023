"""fp64 references of the dense kernels of the SASRec / TIGER training step - the linear GEMM epilogues (csrc/tc_gemm.cuh), the
weight-gradient GEMM (csrc/tc_tn_group.cuh), the bias column sums, LayerNorm, RMS norm and the embedding gather / scatter
(csrc/rowwise.cuh) - that know where the kernels round, numpy restatements of the two fixed summation orders of the embedding
backward, and the checks with their allowances.

Each reference takes the kernel's own inputs (and, where a kernel reads one of its own earlier outputs, that output: the bf16 z
the activation is applied to, the saved LayerNorm / RMS statistics of the backward) and computes in exact fp64.  The rounding of
the kernels is bounded per element, from the magnitudes of the terms an output sums; a check divides the error by that allowance.
Where the operands are small integers times powers of two every product, partial sum and fp32 output is exact, so a kernel must
equal the fp64 value bit for bit whatever its summation order, and a bf16 output must equal its round-to-nearest-even.

Where the kernels round (C = 2^-24 is the fp32 unit roundoff, U = 2^-8 half a bf16 ulp, relative):
  linear forward (TcEpiBiasAct)   z = bf16(acc + bias): the fp32 wgmma sum of K bf16 products, the bias add, one RNE rounding.
                                  a = bf16(dropout(ACT(z))): ACT of the ROUNDED z (bf16_round), then the fp32 keep scale, one RNE
                                  rounding.  ReLU is exact, so a is restated bit for bit from the kernel's z ("a_exact"); SiLU
                                  uses __expf and rcp.approx, bounded by 2^-18 |z| (1 + |z|).
  linear residual (TcEpiBiasResidual)  y = (res + dropout(acc + bias)) * row_scale, fp32 throughout.
  linear backward                 dx = dy W (+ res) (gemm_nn_f32, fp32), dW = dy^T x (per k-split tile sums, then the splits in
                                  order, one add), db = colsum(dy) (per-CTA partials, then det_finish in order).  The fp32 sums get
                                  ACC = 2^-23 per term of sum |terms| (as test_linear_dact_bwd_vs_fp64); over dW's 25,600 tokens
                                  that bound is too loose to see a lost k-split, which the exact operands catch instead.
  LayerNorm (ln_fwd_kernel)       two-pass: mean = sum x / D, var = sum (x - mean)^2 / D in fp32, rstd = rsqrtf(var + eps),
                                  y = (x - mean) rstd g + b -> bf16 and / or fp32.  A row sum takes D / 32 sequential terms per
                                  lane and a 5-level butterfly (DEPTH).  A row with |mean| >> std loses nothing but the rounding of
                                  the mean, which the allowance carries as DEPTH C mean|x|; a one-pass variance loses mean^2 C.
  LayerNorm backward              from the kernel's saved (mean, rstd): xh = (x - mean) rstd, gg = dy g, dx = rstd (gg - mean(gg)
                                  - xh mean(gg xh)) (+ res); dg = sum dy xh, db = sum dy over rows (per warp, per CTA, det_finish).
  RMS norm                        r = rsqrtf(sum x^2 / D + eps), y = w (x r); backward from the saved r: dx = r (gg - xh mean(gg xh))
                                  (+ res), dw = sum dy xh.
  embedding forward               x = dropout(E[id] scale (+ pos[t % L])), times 0 on id 0 when mask_pad_rows: the product and the
                                  add may fuse, so 3 C of the terms.  With scale 1 and p in {0, 0.5} it is exact.
  embedding backward              dE[id] += sum of scale dropmask(dx[t]) over the tokens of id (id 0 never), dpos[l] += sum over b
                                  of dropmask(dx[b L + l]) (id-0 tokens left out when mask_pad_rows); both in fixed fp32 orders
                                  that `embed_dE_fixed_order` / `embed_dpos_fixed_order` restate.

Dropout masks are attention_reference.drop_mask with the token index as row key; the embedding's site is SITE_EMBED.
"""
import math

import numpy as np
import torch

from tests.attention_reference import U, drop_mask, keep_scale

C = 2.0 ** -24                 # fp32 unit roundoff
ACC = 2.0 ** -23               # per-term allowance of an fp32 accumulation
SILU_SLACK = 2.0 ** -18        # __expf + rcp.approx in sigmoidf_fast, times |z| (1 + |z|)
RSQRT = 2.0 ** -22             # rsqrtf: 2 ulp
SITE_EMBED = 250               # csrc/api.cu

# ---- tolerances on the worst ratio |got - ref| / allowance.  Every allowance here is derived (a bound, not a measurement), so
#      the tolerance is 1; tests/test_dense_reference_cpu.py checks that each mutant of what a check guards fails it.
TOL = 1.0


def keep(rows, ncols, p, seed, site, device="cpu"):
    """[len(rows), ncols] fp64 keep-scale matrix of Dropout::apply: 0 where dropped, the fp32 keep scale elsewhere."""
    d = drop_mask(np.asarray(rows), ncols, p, seed, site)
    return torch.from_numpy(np.where(d, 0.0, keep_scale(p)[1])).to(device)


def rne_bf16(x):
    """bf16 round-to-nearest-even of an fp64 tensor whose values are exact in fp32 (so the conversion through fp32 is exact)."""
    f = x.float()
    assert torch.equal(f.double(), x.double()), "value not exact in fp32"
    return f.bfloat16()


# ------------------------------------------------------------------------------------------------ linear
def linear_forward(x, w, bias, act=0, z_kernel=None, p=0.0, seed=0, site=0):
    """x [T, K] bf16, w [N, K] bf16, bias [N] fp32.  -> "z" = acc + bias (fp64) with allowance "a_z"; with act and the kernel's bf16
    z: "a" = ACT(z_kernel) keep with "a_a", and for ReLU "a_exact", the kernel's bf16 result restated (fmaxf, one fp32 product with
    the keep scale, RNE)."""
    X, W, b = x.double(), w.double(), bias.double()
    T, K = X.shape
    z = X @ W.T + b
    mag = X.abs() @ W.abs().T
    r = {"z": z, "a_z": U * z.abs() + (1 + U) * (K * ACC * mag + C * z.abs())}
    if act:
        zk = z_kernel.double()
        km = keep(range(T), W.shape[0], p, seed, site, X.device)
        f = zk.clamp_min(0) if act == 2 else zk * torch.sigmoid(zk)
        r["a"] = f * km
        slack = (SILU_SLACK * zk.abs() * (1 + zk.abs())) if act == 1 else C * f.abs()
        r["a_a"] = U * r["a"].abs() + (1 + U) * slack * km
        if act == 2:
            r["a_exact"] = (f.float() * km.float()).bfloat16()
    return r


def linear_residual(x, w, bias, res, row_scale=None, p=0.0, seed=0, site=0):
    """y = (res + dropout(x w^T + bias)) * row_scale, fp32 in the kernel.  -> "y", "a_y"."""
    X, W, b = x.double(), w.double(), bias.double()
    T, K = X.shape
    y0 = X @ W.T + b
    mag = X.abs() @ W.abs().T + b.abs()
    km = keep(range(T), W.shape[0], p, seed, site, X.device)
    s = row_scale.double()[:, None] if row_scale is not None else torch.ones(T, 1, dtype=torch.float64, device=X.device)
    R = res.double()
    y = (R + y0 * km) * s
    a = s.abs() * (km * (K + 2) * ACC * mag + 2 * C * (R.abs() + km * y0.abs())) + C * y.abs()
    return {"y": y, "a_y": a}


def linear_backward(dy, w, x, res=None):
    """dy [T, N] bf16, w [N, K] bf16, x [T, K] bf16, res [T, K] fp32 or None -> "dx", "dw", "db" with allowances."""
    DY, W, X = dy.double(), w.double(), x.double()
    T, N = DY.shape
    dx = DY @ W
    a_dx = N * ACC * (DY.abs() @ W.abs()) + C * dx.abs()
    if res is not None:
        R = res.double()
        dx = dx + R
        a_dx = a_dx + C * (dx.abs() + R.abs())
    dw = DY.T @ X
    db = DY.sum(0)
    return {"dx": dx, "a_dx": a_dx, "dw": dw, "a_dw": T * ACC * (DY.abs().T @ X.abs()), "db": db, "a_db": T * ACC * DY.abs().sum(0)}


# ------------------------------------------------------------------------------------------------ norms
def _depth(D):
    return D // 32 + 8         # a lane's D / 32 terms, the 5-level butterfly, the division, and a little slack


def layernorm_forward(x, g, b, eps):
    """x [T, D] fp32.  -> "y" (fp64, the value both the bf16 and the fp32 output approximate) with allowances "a_y32" (fp32 output)
    and "a_y16" (bf16 output), "mean" / "rstd" with "a_mean" / "a_rstd"."""
    X, G, Bb = x.double(), g.double(), b.double()
    D = X.shape[1]
    k = _depth(D)
    mean = X.mean(1, keepdim=True)
    xc = X - mean
    var = (xc * xc).mean(1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xh = xc * rstd
    y = xh * G + Bb
    e_mean = k * C * X.abs().mean(1, keepdim=True)
    e_rstd = (e_mean * xc.abs().mean(1, keepdim=True) + k * C * var) / (var + eps) + RSQRT          # relative
    a32 = G.abs() * rstd * (e_mean + C * xc.abs()) + (G * xh).abs() * e_rstd + 3 * C * ((G * xh).abs() + Bb.abs())
    return {"y": y, "a_y32": a32, "a_y16": U * y.abs() + (1 + U) * a32, "mean": mean[:, 0], "a_mean": e_mean[:, 0],
            "rstd": rstd[:, 0], "a_rstd": (e_rstd * rstd)[:, 0]}


def layernorm_backward(dy, x, stats, g, res=None):
    """From the kernel's saved stats [T, 2] = (mean, rstd).  -> "dx", "dg", "db" with allowances."""
    DY, X, G = dy.double(), x.double(), g.double()
    st = stats.double()
    m, r = st[:, 0:1], st[:, 1:2]
    T, D = X.shape
    k = _depth(D)
    xh = (X - m) * r
    gg = DY * G
    sa, sb = gg.mean(1, keepdim=True), (gg * xh).mean(1, keepdim=True)
    dx = r * (gg - sa - xh * sb)
    e_xh = 2 * C * (xh.abs() + r * X.abs())      # x - mean carries the rounding of x's own magnitude
    e_sa = k * C * gg.abs().mean(1, keepdim=True)
    e_sb = k * C * (gg * xh).abs().mean(1, keepdim=True) + (gg.abs() * e_xh).mean(1, keepdim=True)
    a_dx = r * (C * gg.abs() + e_sa + xh.abs() * e_sb + e_xh * sb.abs() + 3 * C * (gg.abs() + sa.abs() + (xh * sb).abs())) + C * dx.abs()
    if res is not None:
        R = res.double()
        dx = dx + R
        a_dx = a_dx + C * dx.abs()
    return {"dx": dx, "a_dx": a_dx, "dg": (DY * xh).sum(0), "a_dg": T * ACC * (DY.abs() * (xh.abs() + e_xh)).sum(0),
            "db": DY.sum(0), "a_db": T * ACC * DY.abs().sum(0)}


def rmsnorm_forward(x, w, eps):
    """x [T, D] fp32 -> "y" with "a_y32" / "a_y16", "rstd" with "a_rstd"."""
    X, W = x.double(), w.double()
    D = X.shape[1]
    k = _depth(D)
    r = 1.0 / torch.sqrt((X * X).mean(1, keepdim=True) + eps)
    y = W * (X * r)
    e_r = k * C + RSQRT                                         # relative: the sum of squares has no cancellation
    a32 = y.abs() * (e_r + 3 * C)
    return {"y": y, "a_y32": a32, "a_y16": U * y.abs() + (1 + U) * a32, "rstd": r[:, 0], "a_rstd": (e_r * r)[:, 0]}


def rmsnorm_backward(dy, x, rstd, w, res=None):
    """From the kernel's saved rstd [T].  -> "dx", "dw" with allowances."""
    DY, X, W = dy.double(), x.double(), w.double()
    r = rstd.double()[:, None]
    T, D = X.shape
    k = _depth(D)
    xh = X * r
    gg = DY * W
    sb = (gg * xh).mean(1, keepdim=True)
    dx = r * (gg - xh * sb)
    e_sb = (k + 2) * C * (gg * xh).abs().mean(1, keepdim=True)
    a_dx = r * (C * gg.abs() + xh.abs() * e_sb + 4 * C * (gg.abs() + (xh * sb).abs())) + C * dx.abs()
    if res is not None:
        dx = dx + res.double()
        a_dx = a_dx + C * dx.abs()
    return {"dx": dx, "a_dx": a_dx, "dw": (DY * xh).sum(0), "a_dw": T * ACC * (DY.abs() * xh.abs()).sum(0)}


# ------------------------------------------------------------------------------------------------ embedding
def embed_forward(ids, E, pos, L, scale, mask_pad_rows, p=0.0, seed=0):
    """On the CPU.  ids [B, L] int64, E [V, D], pos [>= L, D] or None.  -> "x" [T, D] with "a_x", "pad" [T] bool."""
    idf = ids.reshape(-1).cpu()
    T = idf.numel()
    D = E.shape[1]
    e = E.double().cpu()[idf] * float(np.float32(scale))
    mag = e.abs()
    if pos is not None:
        pp = pos.double().cpu()[torch.arange(T) % L]
        e = e + pp
        mag = mag + pp.abs()
    km = keep(range(T), D, p, seed, SITE_EMBED)
    live = ~((idf == 0) & bool(mask_pad_rows))
    x = e * km * live[:, None]
    return {"x": x, "a_x": 3 * C * mag * km * live[:, None], "pad": idf == 0}


def embed_backward(ids, dx, L, V, P, scale, mask_pad_rows, p=0.0, seed=0, dE0=None, dpos0=None):
    """On the CPU.  dx [T, D] fp32; V table rows, P position rows (0: no position table).  -> "dE" [V, D], "dpos" [P, D] (the initial sinks
    dE0 / dpos0 added) with allowances."""
    idf = ids.reshape(-1).cpu()
    T = idf.numel()
    D = dx.shape[1]
    km = keep(range(T), D, p, seed, SITE_EMBED)
    t = dx.double().cpu() * km
    te = t * float(np.float32(scale))
    te[idf == 0] = 0                                          # row 0 of the table never takes a gradient
    dE = torch.zeros(V, D, dtype=torch.float64).index_add_(0, idf, te)
    magE = torch.zeros(V, D, dtype=torch.float64).index_add_(0, idf, te.abs())
    n = torch.bincount(idf, minlength=V).double()[:, None]
    aE = (n + n / 32 + 36) * C * magE
    if dE0 is not None:
        dE = dE + dE0.double().cpu()
    r = {"dE": dE, "a_dE": aE + C * dE.abs()}
    if P:
        tp = t.clone()
        if mask_pad_rows:
            tp[idf == 0] = 0
        l = torch.arange(T) % L
        dpos = torch.zeros(P, D, dtype=torch.float64).index_add_(0, l, tp)
        magp = torch.zeros(P, D, dtype=torch.float64).index_add_(0, l, tp.abs())
        if dpos0 is not None:
            dpos = dpos + dpos0.double().cpu()
        r.update(dpos=dpos, a_dpos=(T // L + 2) * C * magp + C * dpos.abs())
    return r


def embed_dE_fixed_order(ids, dx, dE0):
    """numpy fp32 restatement of embed_bwd_piece_kernel + embed_bwd_run_kernel at scale 1 and p = 0: the tokens sorted by id (stable)
    are cut into pieces of 32 positions; inside a piece each id's tokens are summed in order, then a run's piece sums are added in
    piece order, and that total is added to dE0[id] once.  Id 0 is skipped."""
    idf = ids.reshape(-1).cpu().numpy()
    g = dx.float().cpu().numpy()
    dE = dE0.float().cpu().numpy().copy()
    order = np.argsort(idf, kind="stable")
    sid = idf[order]
    T = len(order)
    starts = np.flatnonzero(np.r_[True, sid[1:] != sid[:-1]])
    ends = np.r_[starts[1:], T]
    for p0, p1 in zip(starts, ends):
        if sid[p0] == 0:
            continue
        cuts = list(range(p0, p1, 32)) if p0 % 32 == 0 else [p0] + list(range((p0 // 32 + 1) * 32, p1, 32))
        seg = [np.cumsum(g[order[a:min(b, p1)]], axis=0, dtype=np.float32)[-1] for a, b in zip(cuts, cuts[1:] + [p1])]
        total = np.cumsum(np.stack(seg), axis=0, dtype=np.float32)[-1]
        dE[sid[p0]] = dE[sid[p0]] + total
    return torch.from_numpy(dE)


def embed_dpos_fixed_order(ids, dx, L, mask_pad_rows, dpos0):
    """numpy fp32 restatement of embed_bwd_pos_kernel at p = 0: dpos0[l] + the sum over b = 0 .. B-1, in ascending b, of
    dx[b L + l] (tokens with id 0 left out when mask_pad_rows)."""
    idf = ids.reshape(-1).cpu().numpy()
    g = dx.float().cpu().numpy()
    T, D = g.shape
    B = T // L
    s = np.zeros((L, D), dtype=np.float32)
    for b in range(B):
        v = g[b * L:(b + 1) * L]
        live = ~((idf[b * L:(b + 1) * L] == 0) & bool(mask_pad_rows))
        s = np.where(live[:, None], s + v, s)
    out = dpos0.float().cpu().numpy().copy()
    out[:L] = out[:L] + s
    return torch.from_numpy(out)


# ------------------------------------------------------------------------------------------------ checks
def worst(got, ref, allow):
    """max over the elements of |got - ref| / allow (0 / 0 counts 0, NaN or Inf gives inf)."""
    d = (got.double().to(ref.device) - ref).abs()
    if not bool(torch.isfinite(d).all()):
        return math.inf
    if d.numel() == 0:
        return 0.0
    r = torch.where(d == 0, torch.zeros_like(d), d / allow.clamp_min(1e-300))
    return r.max().item()


def errors(got, ref, names):
    """{name: worst ratio} over the names present in `got`; ref holds name and "a_" + name."""
    return {n: worst(got[n], ref[n], ref["a_" + n]) for n in names if got.get(n) is not None}


def violations(err, tol=TOL):
    return [f"{n} {w:.3g}" for n, w in err.items() if not w <= tol]


def fmt(err):
    return " ".join(f"{n} {w:.3f}" for n, w in err.items())
