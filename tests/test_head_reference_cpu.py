"""The head checks of tests/head_reference.py catch what they claim to.  An fp32 model of each implementation of the cross-entropy
head - the fused wgmma kernels (ce_rows_kernel / ce_table_kernel: online softmax over 64-class tiles, ex2 with the log2-domain
shift), the stored-logits ce_fwd_bwd_vec_kernel and the scalar ce_fwd_bwd_kernel - must pass them, and each mutant of the fused
model, one plausible defect of a rewritten head, must fail them at the same tolerances."""
import pytest
import torch

from tests.head_reference import CLASS_TILE, L2E, TOL, inv_count, make_case, reference, head_errors, violations

PATHS = ("fused", "vec", "scalar")
CASES = [(70, 64, 65, "small"), (129, 64, 129, "plain"), (130, 128, 2, "plain"), (400, 128, 12102, "plain"), (200, 256, 1203, "plain"),
         (150, 128, 3000, "wide"), (80, 128, 3000, "overflow")]


def _ln_fwd(x, g, b, eps=1e-5):
    """fp32 model of ln_fwd_kernel: (xf bf16, st [T, 2] = mean, rstd)"""
    mean = x.mean(1, keepdim=True)
    rstd = torch.rsqrt(((x - mean) ** 2).mean(1, keepdim=True) + eps)
    return ((x - mean) * rstd * g + b).bfloat16(), torch.cat([mean, rstd], 1)


def _ln_bwd32(dy, x, st, g):
    """fp32 model of ln_bwd_kernel"""
    m, r = st[:, 0:1], st[:, 1:2]
    xh = (x - m) * r
    gg = dy * g
    dx = r * (gg - gg.mean(1, keepdim=True) - xh * (gg * xh).mean(1, keepdim=True))
    return dx, (dy * xh).sum(0), dy.sum(0)


def _to_bf16_rz(g):
    return (g.view(torch.int32) & -65536).view(torch.float32)


def head_model(case, path, mutant=None):
    """fp32 model of grb_head_loss_forward_backward on one implementation; `mutant` plants one defect into the fused model.
    -> ({"loss", "dx", "dg", "db", "dE"}, xf, st)"""
    x, tg = case["x"], case["tg"]
    xf, st = _ln_fwd(x, case["ln_g"], case["ln_b"])
    X, E = xf.float(), case["table"].bfloat16().float()
    T, C = tg.numel(), E.shape[0]
    rows = torch.arange(T)
    valid = tg != 0
    inv = torch.tensor(inv_count(tg), dtype=torch.float32)
    if mutant == "count_plus_one":
        inv = 1.0 / (valid.sum().float() + 1.0)
    ic = torch.where(valid, inv, torch.zeros(()))
    if mutant == "ignored_leak":
        ic[int(torch.nonzero(~valid)[0])] = inv
    S = X @ E.t()
    if path == "fused":
        ncol = C
        if mutant == "pad_logit_zero":                      # the padding of the last class tile enters the softmax as logit 0
            ncol = -(-C // CLASS_TILE) * CLASS_TILE
            S = torch.cat([S, torch.zeros(T, ncol - C)], 1)
        m = torch.full((T,), -float("inf"))
        s = torch.zeros(T)
        for j in range(0, ncol, CLASS_TILE):
            blk = S[:, j:j + CLASS_TILE]
            mn = torch.maximum(m, blk.amax(1))
            s = s * torch.exp2((m - mn) * L2E) + torch.exp2((blk - mn[:, None]) * L2E).sum(1)
            m = mn
        shift = m * L2E + torch.log2(s)
        if mutant == "shift":
            r1, r2 = torch.nonzero(valid)[[3, 11], 0]
            shift[r1] += 1e-3 * L2E
            shift[r2] += 1e-2 * L2E
        tcol = tg.clone()
        if mutant == "target_neighbour":
            r = int(torch.nonzero(valid & (tg < C - 1))[5])
            tcol[r] += 1
        row_loss = (m + torch.log(s) - S[rows, tcol]) * ic
        G = torch.exp2(S * L2E - shift[:, None]) * ic[:, None]
        G = G[:, :C]
        G[rows, tg] -= ic
    elif path == "vec":
        m = S.amax(1)
        e = torch.exp2(S * L2E - (m * L2E)[:, None])
        stot = e.sum(1)
        row_loss = (m + torch.log(stot) - S[rows, tg]) * ic
        G = e * (ic / stot)[:, None]
        G[rows, tg] -= ic
    else:
        m = S.amax(1)
        s = torch.exp(S - m[:, None]).sum(1)
        row_loss = (m + torch.log(s) - S[rows, tg]) * ic
        G = torch.exp(S - m[:, None]) * (1.0 / s)[:, None]
        G[rows, tg] -= 1.0
        G = G * ic[:, None]
    Gb = _to_bf16_rz(G) if mutant == "round_toward_zero" else G.bfloat16().float()
    Gx, Ge = Gb, Gb.clone()
    last = (C - 1) // CLASS_TILE * CLASS_TILE
    if mutant == "dx_last_tile":
        Gx = Gb.clone()
        Gx[:, last:] = 0
    if mutant == "dE_last_tile":
        Ge[:, last:] = 0
    if mutant == "dE_odd_token_tiles":                        # one consumer warpgroup of ce_table_kernel lost
        Ge[(rows // 64) % 2 == 1] = 0
    dxf = Gx @ E
    dE = Ge.t() @ X
    dx, dg, db = _ln_bwd32(dxf, x, st, case["ln_g"])
    return {"loss": row_loss.sum().item(), "dx": dx, "dg": dg, "db": db, "dE": dE}, xf, st


def _errors(case, path, mutant=None):
    got, xf, st = head_model(case, path, mutant)
    ref = reference(case["x"], st, xf, case["ln_g"], case["table"].bfloat16(), case["tg"], chunk=128)
    return head_errors(got, ref, case["tg"])


@pytest.mark.parametrize("T,D,C,kind", CASES)
@pytest.mark.parametrize("path", PATHS)
def test_fp32_model_of_each_kernel_path_passes(path, T, D, C, kind):
    err = _errors(make_case(T, D, C, seed=T * 31 + C, kind=kind), path)
    assert not violations(err), (violations(err), err)


# every mutant runs on the C = 12102 case (last class tile 12096..12101 partial, a fully ignored 128-row token tile), except the
# padding one: its stray columns only carry softmax mass when the logits are within a few nats of each other
MUTANTS = {
    "dx_last_tile": (400, 128, 12102, "plain"),
    "dE_last_tile": (400, 128, 12102, "plain"),
    "dE_odd_token_tiles": (400, 128, 12102, "plain"),
    "shift": (400, 128, 12102, "plain"),
    "target_neighbour": (400, 128, 12102, "plain"),
    "ignored_leak": (400, 128, 12102, "plain"),
    "pad_logit_zero": (70, 64, 65, "small"),
    "count_plus_one": (400, 128, 12102, "plain"),
    "round_toward_zero": (400, 128, 12102, "plain"),
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_mutant_is_rejected(mutant):
    T, D, C, kind = MUTANTS[mutant]
    case = make_case(T, D, C, seed=T * 31 + C, kind=kind)
    assert not violations(_errors(case, "fused")), "the unmutated model must pass on this case"
    err = _errors(case, "fused", mutant)
    assert violations(err), (mutant, err)


def test_case_builder_places_the_edge_targets():
    T, C = 400, 12102
    tg = make_case(T, 128, C, seed=1)["tg"]
    for c in (1, 63, 64, 65, C - 2, C - 1):
        assert (tg == c).any(), c
    assert (tg[128:256] == 0).all() and (tg == 0).sum() > 128
    for r in (0, 63, 64, 127, 256, 319, 320, 383, T - 1):
        assert tg[r] != 0, r
    assert T % 128 != 0                                       # the final token tile is partly past T
    assert set(TOL) >= {"dx frob", "dE frob", "dx row", "dE row", "dx exact", "dE exact", "loss"}
