"""The fp64 reference of the sampled-softmax head (tests/sampled_head_reference.py) against torch autograd on the explicit
formulation: concatenate the target score and the negative scores, mask, F.cross_entropy.  No GPU."""
import pytest
import torch
import torch.nn.functional as F

from tests.sampled_head_reference import make_case, reference

EPS = 1e-5


def _ln_operands(c):
    """What ln_fwd_kernel hands the head: fp32 statistics [T, 2] (mean, rstd) and the bf16 rows."""
    x = c["x"]
    mean = x.mean(1, keepdim=True)
    rstd = torch.rsqrt(x.var(1, unbiased=False, keepdim=True) + EPS)
    xf = ((x - mean) * rstd * c["ln_g"] + c["ln_b"]).bfloat16()
    return torch.cat([mean, rstd], 1), xf


def _autograd(c, xf, tb):
    """loss and gradients of the explicit formulation in fp64; h takes the kernels' bf16 rounding straight through."""
    x = c["x"].double().requires_grad_(True)
    g = c["ln_g"].double().requires_grad_(True)
    b = c["ln_b"].double().requires_grad_(True)
    E = tb.double().requires_grad_(True)
    tg, neg, C = c["tg"], c["neg"], tb.shape[0]
    h = F.layer_norm(x, x.shape[1:], g, b, EPS)
    h = h + (xf.double() - h).detach()
    lq = c["log_q"].double() if c["log_q"] is not None else torch.zeros(C, dtype=torch.float64)
    ok = (neg >= 1) & (neg < C)
    sid = neg.clamp(0, C - 1)
    z = h @ E[sid].t() - lq[sid]
    z = z.masked_fill(~ok[None, :] | (neg[None, :] == tg[:, None]), float("-inf"))
    zt = (h * E[tg]).sum(1) - lq[tg]
    logits = torch.cat([zt[:, None], z], 1)
    valid = tg != 0
    loss = F.cross_entropy(logits[valid], torch.zeros(int(valid.sum()), dtype=torch.long))   # class 0 of the concatenation: the target
    loss.backward()
    return loss.item(), x.grad, g.grad, b.grad, E.grad


def _close(a, r, tol=2e-5):
    return (a - r).norm().item() <= tol * max(r.norm().item(), 1e-30)


@pytest.mark.parametrize("with_log_q", (True, False))
@pytest.mark.parametrize("T,D,C,N", [(37, 64, 50, 70), (130, 128, 20, 5), (9, 64, 300, 1), (64, 128, 7, 129)])
def test_reference_matches_autograd(T, D, C, N, with_log_q):
    """accidental hits, a repeated negative, repeated targets (T > C), ignored tokens and ids outside 1 .. C-1 are all in make_case"""
    c = make_case(T, D, C, N, seed=T + N, with_log_q=with_log_q)
    neg, tg = c["neg"], c["tg"]
    if N > 65:
        assert ((neg < 1) | (neg >= C)).any() and (neg[:, None] == tg[None, :]).any()
        assert neg.unique().numel() < N
    assert (tg == 0).any() and tg[tg != 0].unique().numel() < int((tg != 0).sum())
    st, xf = _ln_operands(c)
    tb = c["table"].bfloat16()
    ref = reference(c["x"], st, xf, c["ln_g"], tb, tg, neg, c["log_q"])
    loss, dx, dg, db, dE = _autograd(c, xf, tb)
    assert abs(ref["loss"] - loss) <= 2e-7 * max(1.0, abs(loss))       # 1 / count is an fp32 number, as ce_count_kernel leaves it
    ex = ref["exact"]
    assert _close(ex["dx"], dx) and _close(ex["dg"], dg) and _close(ex["db"], db) and _close(ex["dE"], dE)
    # the bf16 rounding of G moves the gradients by at most 2^-9 of G, and never the ignored rows
    b16 = ref["bf16"]
    assert _close(b16["dE"], dE, 2 ** -8) and _close(b16["dx"], dx, 2 ** -8)
    assert b16["dx"][tg == 0].abs().max().item() == 0.0


def test_a_constant_added_to_log_q_changes_nothing():
    c = make_case(40, 64, 30, 17, seed=3)
    st, xf = _ln_operands(c)
    tb = c["table"].bfloat16()
    a = reference(c["x"], st, xf, c["ln_g"], tb, c["tg"], c["neg"], c["log_q"])
    b = reference(c["x"], st, xf, c["ln_g"], tb, c["tg"], c["neg"], c["log_q"] + 2.5)
    assert abs(a["loss"] - b["loss"]) <= 1e-6
    for k in ("dx", "dg", "db", "dE"):
        assert _close(b["exact"][k], a["exact"][k], 1e-5)


def test_a_token_whose_every_negative_is_a_hit_has_zero_loss_and_gradient():
    c = make_case(12, 64, 30, 4, seed=5, hits=False)
    c["tg"][:] = torch.tensor([3, 0, 5, 3, 7, 7, 9, 3, 0, 2, 5, 3])
    c["neg"][:] = 3
    st, xf = _ln_operands(c)
    ref = reference(c["x"], st, xf, c["ln_g"], c["table"].bfloat16(), c["tg"], c["neg"], c["log_q"])
    rows = c["tg"] == 3
    assert ref["exact"]["dx"][rows].abs().max().item() == 0.0
    assert ref["exact"]["dx"][c["tg"] == 5].abs().max().item() > 0.0


def test_no_valid_target_gives_nan_loss_and_zero_gradients():
    """the convention of the full head (ce_count_kernel): 1 / count = 0, loss = NaN"""
    c = make_case(8, 64, 30, 4, seed=6)
    c["tg"][:] = 0
    st, xf = _ln_operands(c)
    ref = reference(c["x"], st, xf, c["ln_g"], c["table"].bfloat16(), c["tg"], c["neg"], c["log_q"])
    assert ref["loss"] != ref["loss"]
    assert all(ref["bf16"][k].abs().max().item() == 0.0 for k in ("dx", "dg", "db", "dE"))
