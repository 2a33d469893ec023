"""fp64 reference of the tied-embedding cross-entropy head (grb_head_loss_forward_backward) that rounds where the kernels round,
the cases it is checked on, and the checks with their tolerances.

The head rounds on purpose in three places only:
  1. LN(x) -> bf16 (ln_fwd_kernel, the kernel grb_layernorm_forward launches),
  2. the table -> bf16 (the caller's operand copy),
  3. the softmax gradient G = (softmax - onehot) / count -> bf16, round to nearest even (pack_bf16 in ce_accumulate, or the bf16
     dlogits of the stored-logits path), before the products dX = G E and dE = G^T LN(x).
Everything else is fp32 accumulation.  The reference takes roundings 1 and 2 from the kernels' own operands and applies 3 itself,
all else in fp64, so a correct kernel sits orders of magnitude closer to it than to the exact math.  `exact` (no rounding 3) is
kept as a sanity check that the emulation does not hide a wrong rounding.  Everything runs in row chunks on whichever device the
operands live on, so the benchmark shapes fit.

One effect of rounding 3 the emulation cannot pin down: where the fp64 G lies within a hair of the midpoint between two bf16
values, the kernel's fp32 G may round the other way, a full bf16 ulp of G.  The reference bounds what such flips can do to each
row (`allow_dx`, `allow_dE`), and the dx / dE checks take that much off each row's error before they scale it.  dln_g and dln_b
sum over all rows, where no such per-row bound is tight; their plain Frobenius tolerance covers a flip of one dominant G.
"""
import torch

CLASS_TILE = 64                     # class tile of ce_rows_kernel / ce_table_kernel
L2E = 1.4426950408889634

# ---- tolerances.  Each is ~3x the largest error measured over every case of tests/test_head_exact_gpu.py on an H100 80GB HBM3
#      (700 W power limit); the measured value is quoted beside it.  tests/test_head_reference_cpu.py checks that every mutant of
#      the head it models is rejected at these values.
# fp32 G of the kernels vs the fp64 G: a logit of up to ~60 nats carries ~1e-5 nats of fp32 accumulation error, its product with
# log2(e) and the shift a few more fp32 ulps, ex2.approx ~2 ulp.  A G within this relative distance of a bf16 rounding midpoint
# may round either way (a bound from that arithmetic, not a measurement).
FLIP_BAND = 2e-4
# rows whose norm is below this fraction of the largest row norm of the tensor are scaled by the floor instead.  A row whose
# softmax is nearly one-hot has a gradient ~(1 - p) of the others' and the kernels' fp32 (p - 1) cancels on it: such rows are
# held to the error of the rows that carry the gradient.
ROW_FLOOR = 1e-2
# the loss is compared relative to max(|loss|, LOSS_FLOOR nats): a row's loss is lse - logit[target] in fp32, whose absolute
# error is an ulp of the logits however small the difference
LOSS_FLOOR = 1.0
TOL = {
    # (a) against the G_bf16 emulation: Frobenius norm of the error (each row's flip allowance taken off) over the norm of the
    # tensor.  dx: measured 1.1e-5, in the overflow cases, where dX = (E_hot - E_target) / count lies almost along the direction
    # LayerNorm's backward projects out and its fp32 arithmetic cancels; 5.5e-6 at most elsewhere.  dE: measured 1.6e-6 (cfg2).
    "dx frob": 3e-5,
    "dE frob": 5e-6,
    # dln_g / dln_b: measured 1.7e-4 / 4.0e-4, both at (D, C, T) = (128, 12102, 64), where one row's dominant G sits on a bf16
    # rounding midpoint and flips; 5.3e-5 / 8.5e-5 at most in every other case
    "dg frob": 5e-4,
    "db frob": 1.2e-3,
    # (a) worst row of dx / worst class row of dE, each scaled by its own norm (floored), beyond the flip allowance.  dx: measured
    # 8.4e-5 at C = 2, where most rows are nearly one-hot and the kernels' fp32 (p - 1) cancels; 2.7e-5 at most elsewhere (overflow).
    # dE: measured 1.9e-5 (cfg2).
    "dx row": 2.5e-4,
    "dE row": 6e-5,
    # (b) against G_exact: worst row of |error|_inf / |row|_inf (floored); rounding G to bf16 moves each element by up to 2^-9.
    # Measured 5.1e-3 (dx), 5.3e-3 (dE).
    "dx exact": 1.5e-2,
    "dE exact": 1.5e-2,
    # (c) loss against the fp64 loss, relative to max(|loss|, LOSS_FLOOR): measured 4.7e-7
    "loss": 1.5e-6,
}


# ------------------------------------------------------------------------------------------------ cases
def special_classes(C):
    """Classes every case puts a target on: both sides of the first class-tile edges and the last two classes (the last partial
    class tile when C % 64 != 0), in the order they are handed out."""
    out = []
    for c in (C - 1, 1, 64, 63, 65, C - 2):
        if 1 <= c < C and c not in out:
            out.append(c)
    return out


def make_case(T, D, C, seed, kind="plain"):
    """x [T, D], ln_g, ln_b [D], table [C, D] fp32 and targets [T] int64 (0 = ignored), on the CPU.

    kind: "plain" (table std 0.5: logits ~ N(0, 32)), "small" (table std 0.05: logits within a few nats, so stray padding
    columns would carry real softmax mass), "wide" (logits over +-60 nats, the largest ones in classes far from the first
    tiles) or "overflow" (one class ~190 nats above every other logit of every row, and never the target).

    Targets: ~20 % of the rows ignored; rows 128..255 all ignored when T >= 385 (a fully ignored 128-row token tile); the special
    classes sit on the first and last rows of 64- and 128-row token tiles (rows 0, 63, 64, 127, 256, 319, 320, 383, T - 1)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, D, generator=g)
    ln_g = 1 + 0.1 * torch.randn(D, generator=g)
    ln_b = 0.1 * torch.randn(D, generator=g)
    std = {"plain": 0.5, "small": 0.05, "wide": 1.5, "overflow": 0.005}[kind]
    table = std * torch.randn(C, D, generator=g)
    tg = torch.randint(1, C, (T,), generator=g)
    tg[torch.rand(T, generator=g) < 0.2] = 0
    if T >= 385:
        tg[128:256] = 0
    hot = None
    if kind == "wide":
        table[int(0.66 * C):int(0.7 * C)] *= 1.6              # |logit| up to ~60, the largest far from the first class tiles
    elif kind == "overflow":
        ln_g = torch.ones(D); ln_b = torch.ones(D)
        hot = int(5 * C / 6)
        table[hot] = 1.5                                      # logit = 1.5 * sum(LN(x)) = 1.5 D: ~190 nats at D = 128
        tg[tg == hot] = 7 if hot != 7 else 8
    rows = [r for r in (0, 63, 64, 127, 256, 319, 320, 383, T - 1) if r < T and not (T >= 385 and 128 <= r < 256)]
    rows = list(dict.fromkeys(rows))
    classes = [c for c in special_classes(C) if c != hot]
    for r in rows[len(classes):]:
        if tg[r] == 0:
            tg[r] = 1 + (r * 7919) % (C - 1)
    for i, c in enumerate(classes):
        if i < len(rows):
            tg[rows[i]] = c
        else:                                                 # fewer edge rows than classes: any other valid row
            free = [r for r in range(T) if r not in rows and tg[r] != 0 and int(tg[r]) not in classes]
            if free:
                tg[free[(i * 7919) % len(free)]] = c
    return {"x": x, "ln_g": ln_g, "ln_b": ln_b, "table": table, "tg": tg}


# ------------------------------------------------------------------------------------------------ reference
def bf16_rne(g):
    """fp64 -> fp32 -> bf16 (round to nearest even, as pack_bf16) -> fp64"""
    return g.float().bfloat16().double()


def flip_ulp(g):
    """|bf16 ulp of g| where g lies within FLIP_BAND (relative) of a bf16 rounding midpoint, else 0."""
    bits = g.float().view(torch.int32) & -65536
    lo = bits.view(torch.float32).double()                      # g rounded toward zero
    hi = (bits + 65536).view(torch.float32).double()            # the next bf16 away from zero
    amb = (g - 0.5 * (lo + hi)).abs() <= FLIP_BAND * g.abs()
    return torch.where(amb, (hi - lo).abs(), torch.zeros_like(g))


def inv_count(tg):
    """1 / #(targets != 0) in fp32, as ce_count_kernel computes it (0 when no target is valid)."""
    n = int((tg != 0).sum())
    return float(torch.ones((), dtype=torch.float32) / n) if n else 0.0


def ln_backward64(dy, x, st, g):
    """fp64 LayerNorm backward from the forward's saved fp32 mean / rstd (the statistics ln_bwd_kernel reads)."""
    m, r = st[:, 0:1].double(), st[:, 1:2].double()
    xh = (x.double() - m) * r
    gg = dy * g.double()
    dx = r * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True))
    return dx, (dy * xh).sum(0), dy.sum(0)


def reference(x, st, xf, ln_g, table_bf16, tg, chunk=2048):
    """x [T, D] fp32, st [T, 2] (mean, rstd) and xf [T, D] bf16 from ln_fwd_kernel, ln_g [D], table_bf16 [C, D], tg [T] int64.

    -> {"loss": fp64 mean CE over the valid rows (ignore_index = 0),
        "bf16" / "exact": {"dx", "dg", "db", "dE"} in fp64 from G rounded to bf16 / unrounded,
        "allow_dx" [T], "allow_dE" [C]: the most a flip of a near-midpoint bf16 rounding of G can move each row's norm}"""
    T, D = x.shape
    C = table_bf16.shape[0]
    dev, f64 = x.device, torch.float64
    E = table_bf16.double()
    Ea = E.abs()
    tg = tg.reshape(-1)
    inv = inv_count(tg)
    res = {v: {"dxf": torch.empty(T, D, dtype=f64, device=dev), "dE": torch.zeros(C, D, dtype=f64, device=dev)} for v in ("bf16", "exact")}
    allow_dxf = torch.empty(T, D, dtype=f64, device=dev)
    allow_dE = torch.zeros(C, D, dtype=f64, device=dev)
    loss = torch.zeros((), dtype=f64, device=dev)
    for r0 in range(0, T, chunk):
        r1 = min(T, r0 + chunk)
        X = xf[r0:r1].double()
        t = tg[r0:r1]
        w = (t != 0).double() * inv
        rows = torch.arange(r1 - r0, device=dev)
        S = X @ E.t()
        lse = torch.logsumexp(S, 1)
        loss += ((lse - S[rows, t]) * (t != 0)).sum()
        G = torch.exp(S.sub_(lse[:, None]))
        del S
        G[rows, t] -= 1.0
        G.mul_(w[:, None])
        for name, Gv in (("exact", G), ("bf16", bf16_rne(G))):
            res[name]["dxf"][r0:r1] = Gv @ E
            res[name]["dE"] += Gv.t() @ X
        F = flip_ulp(G)
        del G
        allow_dxf[r0:r1] = F @ Ea
        allow_dE += F.t() @ X.abs()
    out = {"loss": (loss * inv).item() if inv else float("nan")}
    for name in ("bf16", "exact"):
        dx, dg, db = ln_backward64(res[name]["dxf"], x, st, ln_g)
        out[name] = {"dx": dx, "dg": dg, "db": db, "dE": res[name]["dE"]}
    # dx = rstd * P(g * dxf) with P a projection (norm <= 1): a flip moving dxf by at most allow_dxf moves dx by at most this much
    out["allow_dx"] = st[:, 1].double() * (allow_dxf * ln_g.double().abs()).norm(dim=1)
    out["allow_dE"] = allow_dE.norm(dim=1)
    return out


# ------------------------------------------------------------------------------------------------ checks
def _frob(a, r, allow=None):
    """|a - r|_F / |r|_F; with `allow` [rows], each row's error norm first loses its flip allowance"""
    d = a.double() - r
    e = d.norm().item() if allow is None else (d.norm(dim=1) - allow).clamp_min(0.0).norm().item()
    n = r.norm().item()
    return e / n if n > 0 else e


def _worst_row(a, r, allow=None):
    """max over rows of (|a_r - r_r|_2 - allow_r)+ / max(|r_r|_2, ROW_FLOOR * max_r |r_r|_2)"""
    d = (a.double() - r).norm(dim=1)
    if allow is not None:
        d = (d - allow).clamp_min(0.0)
    n = r.norm(dim=1)
    floor = max(ROW_FLOOR * n.max().item(), 1e-30)
    return (d / n.clamp_min(floor)).max().item() if d.numel() else 0.0


def _worst_row_inf(a, r):
    """max over rows of |a_r - r_r|_inf / max(|r_r|_inf, ROW_FLOOR * max |r|)"""
    d = (a.double() - r).abs().amax(1)
    n = r.abs().amax(1)
    floor = max(ROW_FLOOR * n.max().item(), 1e-30)
    return (d / n.clamp_min(floor)).max().item() if d.numel() else 0.0


def head_errors(got, ref, tg):
    """got: {"loss": float, "dx", "dg", "db", "dE"} of the kernels (fp32, on ref's device); ref: reference(...).
    -> {check name: measured error} for every key of TOL, plus "ignored dx": max |dx| over the rows with target 0."""
    b, ex = ref["bf16"], ref["exact"]
    e = {"dx frob": _frob(got["dx"], b["dx"], ref["allow_dx"]), "dE frob": _frob(got["dE"], b["dE"], ref["allow_dE"])}
    e.update({f"{k} frob": _frob(got[k], b[k]) for k in ("dg", "db")})
    e["dx row"] = _worst_row(got["dx"], b["dx"], ref["allow_dx"])
    e["dE row"] = _worst_row(got["dE"], b["dE"], ref["allow_dE"])
    e["dx exact"] = _worst_row_inf(got["dx"], ex["dx"])
    e["dE exact"] = _worst_row_inf(got["dE"], ex["dE"])
    e["loss"] = abs(got["loss"] - ref["loss"]) / max(abs(ref["loss"]), LOSS_FLOOR)
    ign = tg.reshape(-1) == 0
    e["ignored dx"] = got["dx"][ign].abs().max().item() if bool(ign.any()) else 0.0
    return e


def violations(err, tol=TOL):
    """Names of the checks the measured errors fail (NaN fails every check; ignored rows must get exactly zero dx)."""
    bad = [k for k, v in tol.items() if not (err[k] <= v)]
    if not (err["ignored dx"] == 0.0):
        bad.append("ignored dx")
    return bad


def format_table(title, err):
    keys = list(TOL) + ["ignored dx"]
    head = "| case | " + " | ".join(keys) + " |"
    line = f"| {title} | " + " | ".join(f"{err[k]:.2e}" for k in keys) + " |"
    return head, line
