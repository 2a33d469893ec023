"""fp64 reference of the sampled-softmax head (grb_head_sampled_loss_forward_backward) that rounds where the kernels round, and the
cases it is checked on.

The kernels round on purpose in three places, the same three as the full head (tests/head_reference.py): LN(x) -> bf16, the table
-> bf16, and the negatives' softmax gradient G = softmax / count -> bf16 before the products dH = G Es and dEs = G^T H.  The
target's own gradient g_tgt = (p_tgt - 1) / count stays fp32.  The reference takes the first two roundings from the kernels' own
operands and applies the third itself, all else in fp64; `exact` has no third rounding.  The flip allowance of head_reference
(a G within FLIP_BAND of a bf16 rounding midpoint may round either way) is carried over unchanged, and so are its error measures
and tolerances (head_errors, violations, TOL)."""
import torch

from tests.head_reference import bf16_rne, flip_ulp, inv_count, ln_backward64

CLASS_TILE = 64                     # class tile of sce_rows_kernel / sce_table_kernel


def make_case(T, D, C, N, seed, *, with_log_q=True, hits=True):
    """x [T, D], ln_g, ln_b [D], table [C, D] fp32, targets [T] (0 = ignored, ~20 %), negatives [N] and log_q [C] (or None), on the
    CPU.  With `hits` the negatives carry what the head must get right: a repeated id (two classes), ids outside 1 .. C-1 (0, C, a
    negative number: never scored), and the targets of rows 0 and T - 1 (accidental hits); targets repeat whenever T > C."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, D, generator=g)
    ln_g = 1 + 0.1 * torch.randn(D, generator=g)
    ln_b = 0.1 * torch.randn(D, generator=g)
    table = 0.3 * torch.randn(C, D, generator=g)
    tg = torch.randint(1, C, (T,), generator=g)
    tg[torch.rand(T, generator=g) < 0.2] = 0
    if T >= 385:
        tg[128:256] = 0                                       # a fully ignored 128-row token tile
    if T > 2:
        tg[T - 1] = tg[0] if tg[0] != 0 else 1                # a repeated target
        tg[0] = tg[T - 1]
    neg = torch.randint(1, C, (N,), generator=g)
    if hits:
        special = [int(tg[0]), int(tg[T - 1]), 0, C, -3, int(neg[0])]
        slots = [N - 1, 0, 1, 63, 64, 65]
        for s, v in zip(slots, special):
            if 0 <= s < N and (N > 2 or v >= 1):
                neg[s] = v
    log_q = None
    if with_log_q:
        freq = torch.rand(C, generator=g) ** 3 + 1e-3         # a skewed proposal
        log_q = torch.log(freq / freq.sum()).float()
    return {"x": x, "ln_g": ln_g, "ln_b": ln_b, "table": table, "tg": tg, "neg": neg, "log_q": log_q}


def scores(xf, table_bf16, tg, neg, log_q):
    """fp64 corrected scores: z_tgt [T], Z [T, N] (-inf where masked), the checked negative ids (0 where never scored)."""
    C = table_bf16.shape[0]
    E, X = table_bf16.double(), xf.double()
    lq = log_q.double() if log_q is not None else torch.zeros(C, dtype=torch.float64, device=X.device)
    ok = (neg >= 1) & (neg < C)
    sid = torch.where(ok, neg, torch.zeros_like(neg))
    Z = X @ E[sid].t() - lq[sid][None, :]
    Z = Z.masked_fill(~ok[None, :], float("-inf")).masked_fill(neg[None, :] == tg[:, None], float("-inf"))
    zt = (X * E[tg]).sum(1) - lq[tg]
    return zt, Z, sid


def reference(x, st, xf, ln_g, table_bf16, tg, neg, log_q):
    """x [T, D] fp32, st [T, 2] (mean, rstd) and xf [T, D] bf16 from ln_fwd_kernel, table_bf16 [C, D], tg [T], neg [N], log_q [C] | None
    -> the dict of head_reference.reference: loss, "bf16" / "exact" gradients, allow_dx, allow_dE."""
    C, D = table_bf16.shape
    dev, f64 = x.device, torch.float64
    E, X = table_bf16.double(), xf.double()
    tg = tg.reshape(-1)
    inv = inv_count(tg)
    w = (tg != 0).double() * inv
    zt, Z, sid = scores(xf, table_bf16, tg, neg, log_q)
    lse = torch.logsumexp(torch.cat([zt[:, None], Z], 1), 1)
    loss = ((lse - zt) * (tg != 0)).sum()
    G = torch.exp(Z - lse[:, None]) * w[:, None]
    gt = (torch.exp(zt - lse) - 1.0) * w
    Es = E[sid]
    out = {"loss": (loss * inv).item() if inv else float("nan")}
    for name, Gv in (("exact", G), ("bf16", bf16_rne(G))):
        dxf = Gv @ Es + gt[:, None] * E[tg]
        dE = torch.zeros(C, D, dtype=f64, device=dev)
        dE.index_add_(0, sid, Gv.t() @ X)                     # never-scored negatives carry G = 0 into row 0
        dE.index_add_(0, tg, gt[:, None] * X)                 # ignored tokens carry g_tgt = 0 into row 0
        dx, dg, db = ln_backward64(dxf, x, st, ln_g)
        out[name] = {"dx": dx, "dg": dg, "db": db, "dE": dE}
    F = flip_ulp(G)
    allow_dE = torch.zeros(C, D, dtype=f64, device=dev).index_add_(0, sid, F.t() @ X.abs())
    out["allow_dx"] = st[:, 1].double() * ((F @ Es.abs()) * ln_g.double().abs()).norm(dim=1)
    out["allow_dE"] = allow_dE.norm(dim=1)
    return out
