"""COBRA's autograd Functions under dropout against fp64 references, on the H100.

Each of genrec_b200.cobra's _LayerNormFn, _SegLnMeanFn, _L2NormFn, _InfoNceFn, _LinearF32Fn, _FfnFn and _MhaFn (packed at head dim 96,
padded and causal with key padding at head dims 32 and 64) runs forward and backward on seeded inputs, and every stage is compared
with its fp64 reference (tests/cobra_stage_reference.py, tests/dense_reference.py, tests/attention_reference.py) on the kernel's own
inputs to that stage.  The forward intermediates come from grad_fn.saved_tensors / grad_fn.cfg, the rest from a spy on
genrec_b200.functional and on the attention core backward.  dy is small integers / 64, so the masked bf16 casts are exact and
checked bit for bit; the dropout masks are restated from (seed, site), so a backward that pairs a stage with another stage's mask
fails here.  The shapes sit at the kernels' edges: rows around a CTA's 8 warps and past the grid-stride wraps, widths 64 to 768,
text lengths around the core's 32-row tiles on both sides of its atomics / partials switch (longest text 64), InfoNCE batches of
1 to 257 rows with every user grouping, and catalogs whose texts x heads exceed the core's 65,535-row grid.

Part B: Cobra.forward and backward at p = 0.1 and 0.3, every dropout included, against tests/cobra_reference.py in fp64 on the same
masks, with the restatement under bf16 autocast as the yardstick.

`pytest -s` prints the worst error / allowance of every part A quantity and the yardstick table of every part B step."""
import pytest
import torch

from tests import attention_reference as ar
from tests import cobra_params as cp
from tests import cobra_reference as cr
from tests import cobra_stage_reference as sr
from tests import dense_reference as dr
from tests import hstu_block_reference as hr
from tests.exact_check import (FTZ, Ledger, Spy, _TorchDropout, _cid, _dy, _packed_core_ref, _seeded, _sms,
                                autocast_yardstick)

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
PS = [0.0, 0.1, 0.3]
EPS = 1e-5                                            # nn.LayerNorm
SEED = 0x2F6B_1D3C_5A79_4E81                          # a 62-bit dropout seed, as Cobra._seed draws
LEDGER = Ledger("worst error / allowance per quantity of the COBRA stages (dense tolerance 1, attention core: attention_reference.TOL):",
                width=18, floor=FTZ)
_error_table = LEDGER.fixture()
_check = LEDGER.check


def _spy(monkeypatch):
    """the functional calls made while it is active"""
    from genrec_b200 import cobra
    from genrec_b200 import functional as Fn
    return Spy(monkeypatch, {Fn: ("cast_rows_bf16", "linear_bwd", "linear_dact_bwd", "infonce_fwd_bwd"),
                             cobra: ("attention_core_bwd", "attention_core_bwd_jagged")})


def _offsets(lens):
    o = [0]
    for n in lens:
        o.append(o[-1] + n)
    return o


# ------------------------------------------------------------------------------------------------ LayerNorm rows
# rows around one CTA's 8 warps, and one past the backward's (3 CTAs per SM) and the forward's (8 per SM) grid-stride wraps
LN_ROWS = ["1", "7", "8", "9", "bwd wrap", "fwd wrap"]
LN_CASES = [(D, R) for D in (192, 384, 768, 64, 128, 256) for R in LN_ROWS]


def _rows(R):
    return {"bwd wrap": 3 * 8 * _sms() + 1, "fwd wrap": 8 * 8 * _sms() + 1}.get(R) or int(R)


@pytest.mark.parametrize("case", LN_CASES, ids=_cid)
def test_layernorm_stage(case):
    from genrec_b200.cobra import _LayerNormFn
    D, R = case
    T = _rows(R)
    x = _seeded((T, D), T + D, 2.0, 0.5).requires_grad_(True)
    g = _seeded((D,), D, 0.1, 1.0).requires_grad_(True)
    b = _seeded((D,), D + 1, 0.1).requires_grad_(True)
    y = _LayerNormFn.apply(x, g, b, EPS)
    xc, st, _ = y.grad_fn.saved_tensors
    dy = _dy((T, D), T)
    y.backward(dy)
    f = dr.layernorm_forward(xc, g.detach(), b.detach(), EPS)
    bw = dr.layernorm_backward(dy, xc, st, g.detach())
    # xh may be formed as x rstd - mean rstd (one fused product): its rounding then scales with |mean| rstd, not |x| rstd.  Over
    # many rows the T ACC sum bound covers it; a single row needs it said
    a_dg = bw["a_dg"] + 2 * dr.C * (dy.double().abs() * (st[:, 0:1].double() * st[:, 1:2].double()).abs()).sum(0)
    _check(_cid(case), [("ln y", y.detach(), f["y"], f["a_y32"]), ("ln mean", st[:, 0], f["mean"], f["a_mean"]),
                        ("ln rstd", st[:, 1], f["rstd"], f["a_rstd"]), ("ln dx", x.grad, bw["dx"], bw["a_dx"]),
                        ("ln dg", g.grad, bw["dg"], a_dg), ("ln db", b.grad, bw["db"], bw["a_db"])])


# ------------------------------------------------------------------------------------------------ pooled LayerNorm mean
SEG_LENS = [0, 1, 7, 8, 9, 17, 128, 512, 0, 3]


@pytest.mark.parametrize("D", [128, 192, 256, 384, 768])
def test_seg_layernorm_mean_stage(D):
    from genrec_b200.cobra import _SegLnMeanFn
    lens = SEG_LENS
    o = _offsets(lens)
    offsets = torch.tensor(o, dtype=torch.int64, device=DEV)
    N, rows = len(lens), o[-1]
    x = _seeded((rows, D), D + 3, 2.0, 0.5).requires_grad_(True)
    g = _seeded((D,), D + 4, 0.1, 1.0).requires_grad_(True)
    b = _seeded((D,), D + 5, 0.1).requires_grad_(True)
    pooled = _SegLnMeanFn.apply(x, g, b, offsets, EPS)
    xc, st, _, _ = pooled.grad_fn.saved_tensors
    dp = _dy((N, D), D + 6)
    pooled.backward(dp)
    f = sr.seg_layernorm_mean_forward(offsets, xc, g.detach(), b.detach(), EPS)
    bw = sr.seg_layernorm_mean_backward(offsets, xc, st, g.detach(), dp)
    empty = f["empty"]
    assert bool(empty.any()) and not bool(pooled.detach()[empty].any()), "a text without rows has a non-zero pooled row"
    _check(f"D{D}", [("pool y", pooled.detach(), f["pooled"], f["a_pooled"]), ("pool mean", st[:rows, 0], f["mean"], f["a_mean"]),
                     ("pool rstd", st[:rows, 1], f["rstd"], f["a_rstd"]), ("pool dx", x.grad, bw["dx"], bw["a_dx"]),
                     ("pool dg", g.grad, bw["dg"], bw["a_dg"]), ("pool db", b.grad, bw["db"], bw["a_db"])])
    # a text without rows adds exactly zero to dg and db: another gradient on those texts alone changes no bit
    from genrec_b200 import functional as Fn
    dp2 = dp.clone()
    dp2[empty] = _dy((int(empty.sum()), D), D + 7) * 37
    _, dg1, db1 = Fn.seg_layernorm_mean_bwd(offsets, xc, st, g.detach().contiguous(), dp.contiguous())
    _, dg2, db2 = Fn.seg_layernorm_mean_bwd(offsets, xc, st, g.detach().contiguous(), dp2.contiguous())
    assert torch.equal(dg1, dg2) and torch.equal(db1, db2), "a text without rows reached dg or db"
    assert torch.equal(dg1, g.grad) and torch.equal(db1, b.grad)


# ------------------------------------------------------------------------------------------------ L2 norm
@pytest.mark.parametrize("case", [(D, R) for D in (128, 384, 768) for R in ("1", "9", "grid wrap")], ids=_cid)
def test_l2norm_stage(case):
    """rows of every scale, a zero row and rows below eps; one past the grid-stride wrap (16 CTAs of 8 warps per SM)"""
    from genrec_b200.cobra import _L2NormFn
    D, R = case
    T = 16 * 8 * _sms() + 1 if R == "grid wrap" else int(R)
    scale = torch.logspace(-3, 3, T, dtype=torch.float64).float().to(DEV)[:, None] if T > 1 else torch.ones(1, 1, device=DEV)
    x = _seeded((T, D), T + D) * scale
    if T > 1:
        x[T // 2] = 0                                                     # n = 0 <= eps: y = 0, dx = dy / eps
        x[T // 3] *= 1e-15                                                # 0 < n < eps
    x.requires_grad_(True)
    y = _L2NormFn.apply(x)
    ys, n = y.grad_fn.saved_tensors
    dy = _dy((T, D), T + 1)
    y.backward(dy)
    f = sr.l2norm_forward(x.detach())
    bw = sr.l2norm_backward(dy, ys, n)
    if T > 1:
        assert not bool(y.detach()[T // 2].any()) and not bool(bw["big"][T // 2]) and not bool(bw["big"][T // 3])
    _check(_cid(case), [("l2 y", y.detach(), f["y"], f["a_y"]), ("l2 norm", n, f["norm"], f["a_norm"]),
                        ("l2 dx", x.grad, bw["dx"], bw["a_dx"])])


# ------------------------------------------------------------------------------------------------ InfoNCE
def _groups(Q, kind):
    """items per user: one user; every user one item; mixed sizes; mixed with one long user last (its range ends at Q)"""
    if kind == "one user":
        return [Q]
    if kind == "singles":
        return [1] * Q
    g = torch.Generator().manual_seed(Q)
    counts, left = [], Q if kind == "mixed" else Q - Q // 2
    while left:
        c = min(int(torch.randint(1, 8, (1,), generator=g)), left)
        counts.append(c)
        left -= c
    return counts if kind == "mixed" else counts + [Q // 2]


NCE_CASES = [(Q, k) for Q in (1, 2, 127, 128, 129, 257) for k in ("one user", "singles", "mixed", "long last")
             if not (Q == 1 and k != "one user")]


@pytest.mark.parametrize("case", NCE_CASES, ids=_cid)
def test_infonce_stage(case, monkeypatch):
    from genrec_b200.cobra import _InfoNceFn
    Q, kind = case
    counts = _groups(Q, kind)
    if kind == "long last" and Q > 1:
        assert counts[-1] == Q // 2 and sum(counts) == Q
    d = 384
    cnt = torch.tensor(counts, device=DEV)
    user = torch.arange(len(counts), device=DEV).repeat_interleave(cnt)
    hi = cnt.cumsum(0)[user]
    lo = hi - cnt[user]
    pred = torch.nn.functional.normalize(_seeded((Q, d), Q + 11), dim=-1).requires_grad_(True)
    gt = torch.nn.functional.normalize(_seeded((Q, d), Q + 12), dim=-1)
    spy = _spy(monkeypatch)
    loss = _InfoNceFn.apply(pred, gt, lo.contiguous(), hi.contiguous(), 1 / 0.2)
    pb, gb, (S, _, _), (lsum, dS) = spy.take("cast_rows_bf16", "cast_rows_bf16", "linear_bwd", "infonce_fwd_bwd")
    dS_saved, gpad = loss.grad_fn.saved_tensors
    Qp = gpad.shape[0]
    assert Qp == (Q + 127) // 128 * 128 and torch.equal(dS_saved, dS)
    assert torch.equal(pb, pred.detach().bfloat16()) and torch.equal(gpad[:Q], gt.bfloat16()) and not bool(gpad[Q:].any())
    loss.backward()
    (dpred, _, _), = spy.take("linear_bwd")
    sf = dr.linear_backward(pb, gpad.t().contiguous(), pb)
    r = sr.infonce_rows(S, Q, lo, hi, 1 / 0.2)
    dp = sr.dpred(dS, gpad, pb)
    assert not bool(dS[r["zero"]].any()), "dS != 0 in a left-out or padding column"
    if bool(r["only_self"].all()):
        assert lsum.item() == 0 and loss.item() == 0, "a row that keeps only itself has a non-zero loss"
    if kind == "one user" and Q > 1:
        assert bool(r["only_self"].all())
    _check(_cid(case), [("nce S", S, sf["dx"], sf["a_dx"]), ("nce loss", loss.detach(), r["loss"], r["a_loss"]),
                        ("nce dS", dS, r["ds"], r["a_ds"]), ("nce dpred", pred.grad, dp["dx"], dp["a_dx"])])


# ------------------------------------------------------------------------------------------------ fp32 linear (proj, heads)
@pytest.mark.parametrize("case", [(K, N, R) for K, N in ((192, 128), (768, 384), (384, 256)) for R in (0, 1, 65, 1000)], ids=_cid)
def test_linear_f32_stage(case, monkeypatch):
    from genrec_b200.cobra import _LinearF32Fn
    K, N, R = case
    x = _seeded((R, K), K + R, 2.0).requires_grad_(True)
    w = _seeded((N, K), N, K ** -0.5).requires_grad_(True)
    b = _seeded((N,), N + 1, 0.5).requires_grad_(True)
    spy = _spy(monkeypatch)
    y = _LinearF32Fn.apply(x, w, b)
    assert y.dtype == torch.float32 and y.shape == (R, N)
    dy = _dy((R, N), R + 2)
    if R == 0:
        y.backward(dy)
        assert not spy.calls and not bool(x.grad.any()) and not bool(w.grad.any()) and not bool(b.grad.any())
        assert w.grad.shape == w.shape and b.grad.shape == b.shape
        return
    xb, (y0, _, _) = spy.take("cast_rows_bf16", "linear_bwd")
    _, wb = y.grad_fn.saved_tensors
    assert torch.equal(xb, x.detach().bfloat16()) and torch.equal(wb, w.detach().bfloat16())
    y.backward(dy)
    dyb, (dx, dw, _) = spy.take("cast_rows_bf16", "linear_bwd")
    assert torch.equal(dyb, dr.rne_bf16(dy.double()))
    f = dr.linear_backward(xb, wb.t().contiguous(), xb)
    yref = f["dx"] + b.detach().double()
    bw = dr.linear_backward(dyb, wb, xb)
    _check(_cid(case), [("f32lin y", y.detach(), yref, f["a_dx"] + dr.C * (yref.abs() + b.detach().double().abs())),
                        ("f32lin dx", x.grad, bw["dx"], bw["a_dx"]), ("f32lin dw", w.grad, bw["dw"], bw["a_dw"]),
                        ("f32lin db", b.grad, bw["db"], bw["a_db"])])


# ------------------------------------------------------------------------------------------------ FFN
# (D, rows): the encoder's widths (192 small, 768 trainer) on packed text rows, the decoder's (384) on B x Li rows
FFN_CASES = [(D, R, p) for D, rows in ((192, (1, 65, 1000)), (768, (64, 1000)), (384, (127, 2048))) for R in rows for p in PS]


@pytest.mark.parametrize("case", FFN_CASES, ids=_cid)
def test_ffn_stage(case, monkeypatch):
    from genrec_b200.cobra import _FfnFn
    D, R, p = case
    Fd = 2048
    site = 16 * 3 + 2
    x = _seeded((R, D), 3 * R + D, 2.0).requires_grad_(True)
    w1 = _seeded((Fd, D), D + 1, D ** -0.5).requires_grad_(True)
    b1 = _seeded((Fd,), D + 2, 0.1).requires_grad_(True)
    w2 = _seeded((D, Fd), D + 3, Fd ** -0.5).requires_grad_(True)
    b2 = _seeded((D,), D + 4, 0.1).requires_grad_(True)
    y = _FfnFn.apply(x, w1, b1, w2, b2, p, p, SEED, site)
    xb, z, h, w1b, w2b = y.grad_fn.saved_tensors
    assert y.grad_fn.cfg == (p, p, SEED, site)
    dy = _dy((R, D), R + 1)
    spy = _spy(monkeypatch)
    y.backward(dy)
    dyb, (_, dw2, db2), dz, (dx, dw1, db1) = spy.take("cast_rows_bf16", "linear_bwd", "linear_dact_bwd", "linear_bwd")
    xc = x.detach()
    f1 = dr.linear_forward(xb, w1b, b1.detach(), 2, z, p, SEED, site)
    f2 = dr.linear_residual(h, w2b, b2.detach(), xc, None, p, SEED, site + 1)
    kh = dr.keep(range(R), Fd, p, SEED, site, DEV)
    ko = dr.keep(range(R), D, p, SEED, site + 1, DEV)
    assert torch.equal(xb, xc.bfloat16())
    assert torch.equal(h, f1["a_exact"]), "h is not RNE(relu(z) keep(site))"
    dead = (kh == 0) | (z.double() <= 0)
    assert not bool(h[dead].any()) and not bool(dz[dead].any()), "h or dz != 0 where keep(site) drops or z <= 0"
    assert torch.equal(dyb, hr.cast_colsum(dy, p, SEED, site + 1)["dyb_exact"]), "dyb is not RNE(keep(site + 1) dy)"
    if p > 0:
        assert bool((kh == 0).any()) and bool((ko == 0).any())
    b2r = dr.linear_backward(dyb, w2b, h)
    dzr = hr.linear_dact_backward(dyb, w2b, z, p, SEED, site, act=2)
    b1r = dr.linear_backward(dz, w1b, xb, res=dy)
    _check(_cid(case), [("ffn z", z, f1["z"], f1["a_z"]), ("ffn h", h, f1["a"], f1["a_a"]), ("ffn y", y.detach(), f2["y"], f2["a_y"]),
                        ("ffn dw2", dw2, b2r["dw"], b2r["a_dw"]), ("ffn db2", db2, b2r["db"], b2r["a_db"]),
                        ("ffn dz", dz, dzr["g"], dzr["a_g"]), ("ffn dx", dx, b1r["dx"], b1r["a_dx"]),
                        ("ffn dw1", dw1, b1r["dw"], b1r["a_dw"]), ("ffn db1", db1, b1r["db"], b1r["a_db"])])
    assert torch.equal(x.grad, dx) and torch.equal(w1.grad, dw1) and torch.equal(w2.grad, dw2)
    assert torch.equal(b1.grad, db1) and torch.equal(b2.grad, db2)


# ------------------------------------------------------------------------------------------------ self-attention
# packed texts at head dim 96 (the encoder: 192 / 2 heads small, 768 / 8 trainer), longest text <= 64 (the backward's atomics)
# and > 64 (its per-query-tile partials, short texts beside long ones); padded causal decoder batches with key padding at head
# dims 64 (128 / 2 small, 384 / 6 trainer) and 32 (128 / 4)
MHA_SHAPES = [
    ("packed", 192, 2, (1, 31, 32, 33, 63, 64)), ("packed", 192, 2, (1, 31, 32, 33, 63, 64, 65, 96, 128, 129)),
    ("packed", 768, 8, (129, 1, 33, 2, 65)), ("packed", 192, 2, (64,)), ("packed", 192, 2, (129,)),
    ("padded", 128, 2, (4, 80)), ("padded", 384, 6, (5, 64)), ("padded", 128, 4, (3, 33)), ("padded", 128, 2, (1, 8)),
]
MHA_CASES = [s + (p,) for s in MHA_SHAPES for p in PS]


def _mid(c):
    f, D, H, shp, p = c
    return f"{f}-D{D}-H{H}-{'x'.join(map(str, shp))}-p{p}"


@pytest.mark.parametrize("case", MHA_CASES, ids=_mid)
def test_mha_stage(case, monkeypatch):
    from genrec_b200.cobra import _MhaFn
    form, D, H, shp, p = case
    packed = form == "packed"
    site = 16 * 2 + 1
    if packed:
        lens = list(shp)
        offs = _offsets(lens)
        offsets = torch.tensor(offs, dtype=torch.int64, device=DEV)
        mx = max(lens)
        x = _seeded((offs[-1], D), D + sum(lens), 2.0)
        key_pad, causal, jag = None, False, (offsets, mx)
    else:
        B, L = shp
        x = _seeded((B, L, D), D + B * L, 2.0)
        n_valid = (torch.arange(B) * 29 % L) + 1                         # right padding, as the interleaved items leave it
        n_valid[0] = L
        key_pad = (torch.arange(L)[None, :] >= n_valid[:, None]).to(torch.uint8).to(DEV)
        causal, jag = True, (None, 0)
    x.requires_grad_(True)
    w_in = _seeded((3 * D, D), D + 1, D ** -0.5).requires_grad_(True)
    b_in = _seeded((3 * D,), D + 2, 0.1).requires_grad_(True)
    w_out = _seeded((D, D), D + 3, D ** -0.5).requires_grad_(True)
    b_out = _seeded((D,), D + 4, 0.1).requires_grad_(True)
    out = _MhaFn.apply(x, w_in, b_in, w_out, b_out, H, p, SEED, site, key_pad, causal, *jag)
    xb, QKV, A, lse, wib, wob, _, _ = out.grad_fn.saved_tensors
    Hc, pc, seed, sc, scale, *_ = out.grad_fn.cfg
    assert (Hc, pc, seed, sc) == (H, p, SEED, site)
    dy = _dy(tuple(out.shape), D + H)
    spy = _spy(monkeypatch)
    out.backward(dy)
    core = "attention_core_bwd_jagged" if packed else "attention_core_bwd"
    dyb, (dA, dwo, _), dAb, (dQ, dK, dV, _), dqkvb, (dx, dwi, _) = spy.take(
        "cast_rows_bf16", "linear_bwd", "cast_rows_bf16", core, "cast_rows_bf16", "linear_bwd")
    flat = lambda t: t.reshape(-1, t.shape[-1])
    case_id = _mid(case)
    Q, K, V = QKV[..., :D], QKV[..., D:2 * D], QKV[..., 2 * D:]
    pin = dr.linear_forward(flat(xb), wib, b_in.detach())
    po = dr.linear_forward(flat(A), wob, b_out.detach())
    items = [("mha QKV", flat(QKV), pin["z"], pin["a_z"]), ("mha out", flat(out.detach()), po["z"], po["a_z"])]
    assert torch.equal(dyb, dr.rne_bf16(dy.double())) and torch.equal(dAb, dA.bfloat16())
    if packed:
        ref = _packed_core_ref(Q, K, V, A, dAb, H, None, offs, 0, scale, p, seed, site)
        got = {"out": A, "dq": dQ, "dk": dK, "dv": dV}
    else:
        ref = ar.t5_reference(Q, K, V, H, None, None, key_pad, causal, scale, dAb, A, p, seed, site)
        got = {"out": A, "dq": dQ, "dk": dK, "dv": dV}
        assert not ar.t5_exact(got, ref, key_pad)
    names = ("out", "dq", "dk", "dv")
    LEDGER.check_core(case_id, ar.errors({k: flat(got[k]) for k in names}, {k: flat(ref[k]) for n in names for k in (n, "a_" + n)}, names),
                      "t5")
    dqkv = torch.cat([dQ.float(), dK, dV], dim=-1)
    assert torch.equal(dqkvb, dqkv.bfloat16())
    bo = dr.linear_backward(flat(dyb), wob, flat(A))
    bi = dr.linear_backward(flat(dqkvb), wib, flat(xb))
    items += [("mha dA", flat(dA), bo["dx"], bo["a_dx"]), ("mha dwo", dwo, bo["dw"], bo["a_dw"]), ("mha dx", flat(x.grad), bi["dx"], bi["a_dx"]),
              ("mha dwi", dwi, bi["dw"], bi["a_dw"]),
              ("mha dbi", b_in.grad, flat(dqkv).double().sum(0), flat(dqkv).shape[0] * dr.ACC * flat(dqkv).double().abs().sum(0)),
              ("mha dbo", b_out.grad, flat(dy).double().sum(0), flat(dy).shape[0] * dr.ACC * flat(dy).double().abs().sum(0))]
    assert torch.equal(w_in.grad, dwi) and torch.equal(w_out.grad, dwo)
    _check(case_id, items)


# ------------------------------------------------------------------------------------------------ a catalog past the core's grid
def test_encode_items_past_the_attention_grid():
    """encode_items under no_grad on 8,200 texts x 8 heads (> 65,535: the split forward grid) at the trainer's shape, against the
    fp64 encoder on a seeded sample of the texts and against the same texts encoded alone"""
    cfg = cp.TRAINER
    from genrec_b200.cobra import MAX_ATTN_ROWS, Cobra
    m = Cobra(**cfg)
    m.load_state_dict(cp.cobra_params(cp.shapes(cfg), 31))
    m = m.to(DEV).eval()
    N, L = 8200, 48
    assert N * cfg["encoder_num_heads"] > MAX_ATTN_ROWS
    g = torch.Generator().manual_seed(32)
    lens = torch.randint(0, L + 1, (N,), generator=g)
    tokens = torch.randint(1, cfg["encoder_vocab_size"], (N, L), generator=g) * (torch.arange(L)[None, :] < lens[:, None])
    with torch.no_grad():
        v = m.encode_items(tokens.to(DEV))
        sample = torch.randperm(N, generator=g)[:64]
        sample = torch.cat([sample, torch.tensor([N - 1])])              # the last text, in the last CTA of the split grid
        alone = m.encode_items(tokens[sample].to(DEV))
        P = {k: t.to(DEV).double() for k, t in cp.cobra_params(cp.shapes(cfg), 31).items() if k.startswith("encoder.")}
        ref = torch.nn.functional.normalize(cr.encode(P, cfg, tokens[sample].to(DEV)), dim=-1)
    live = lens[sample] > 0
    got = v[sample.to(DEV)]
    err = ((got - ref).abs().max() / ref.abs().max()).item()
    # measured 3.7e-3 on an H100 (bf16 operands through one 768-wide encoder layer); the bound is ~2.5x that
    print(f"\nencode_items N={N}: max-norm relative error {err:.3g} against fp64")
    assert err <= 1e-2
    assert torch.allclose(got, alone, rtol=0, atol=1e-5)
    assert bool(live.any()) and bool((lens == 0).any())


# ------------------------------------------------------------------------------------------------ part B: the whole step
def _geometric_items(B, cap, seed):
    """items per user: 2 + a geometric count (mean 3), capped"""
    g = torch.Generator().manual_seed(seed)
    u = torch.rand(B, generator=g).clamp_min(1e-9)
    return tuple(min(cap, 2 + int(v)) for v in (u.log() / torch.tensor(0.75).log()).floor().tolist())


# (shape, p): SMALL on the ragged batch of cobra_small.pt (users of 1, 2, 7 and 20 items); SMALL at B = 256 (2,048 texts, past the
# packing scan's 1,024-text chunks); the trainer's shape at B = 32
STEPS = [("small", 0.1), ("small", 0.3), ("small B=256", 0.1), ("small B=256", 0.3), ("trainer B=32", 0.1)]


@pytest.mark.parametrize("case", STEPS, ids=_cid)
def test_training_step_vs_fp64(case, monkeypatch):
    """Cobra.forward + backward with every dropout at p against the fp64 restatement on the same masks: torch's F.dropout masks
    recorded by a shim, the kernels' restated from the step's two seeds (cobra_reference.kernel_step_masks).  The yardstick is the
    restatement under bf16 autocast (exact_check.autocast_yardstick); the integer metrics match to within the counted
    positions whose top-1 lead is below cobra_reference.MARGIN."""
    from genrec_b200 import cobra
    from tests.util import frob_relerr, relerr
    shape, p = case
    trainer = shape.startswith("trainer")
    cfg = dict(cp.TRAINER if trainer else cp.SMALL, decoder_dropout=p)
    if shape == "small":
        ids, text = cp.batch(cfg, seed=109)
    else:
        B, cap, L = (32, 10, 128) if trainer else (256, 8, 64)
        ids, text = cp.batch(cfg, items=_geometric_items(B, cap, B), text_lens=(1, 37, L), L=L, seed=B + 1)
    B, T, L = text.shape
    params = cp.cobra_params(cp.shapes(cfg), 309 if trainer else 109)
    m = cobra.Cobra(**cfg)
    m.load_state_dict(params)
    for mod in m.modules():                                  # the encoder's too (its dropout is fixed at 0.1)
        if isinstance(mod, torch.nn.Dropout):
            mod.p = p
        if isinstance(mod, torch.nn.MultiheadAttention):
            mod.dropout = p
    m = m.to(DEV).train()
    shim = _TorchDropout()
    monkeypatch.setattr(cobra, "F", shim)
    seeds, draw = [], m._seed
    m._seed = lambda: seeds.append(draw()) or seeds[-1]
    torch.manual_seed(2000 + B + int(10 * p))
    out = m(ids.to(DEV), text.to(DEV))
    out.loss.backward()
    assert len(seeds) == 2 and len(shim.masks) == cfg.get("encoder_n_layers", 1) + 2 * cfg["decoder_n_layers"]
    masks = cr.kernel_step_masks(params, cfg, ids, text, p, seeds, shim.masks, DEV)
    for i, k in enumerate(masks):
        assert bool((k == 0).any()), f"mask {i} {tuple(k.shape)} keeps everything"
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ref, rgrads = cr.step(params, cfg, ids, text, device=DEV, masks=masks)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    ac, agrads = cr.step(params, cfg, ids, text, dtype=torch.float32, device=DEV, masks=masks, autocast=True)
    for k in ("acc_total", "recall_total"):
        assert getattr(out, k).item() == ref[k].item(), k
    near = ref["near"].item()
    for k in ("acc_correct", "recall_correct"):
        assert abs(getattr(out, k).item() - ref[k].item()) <= near, (k, getattr(out, k).item(), ref[k].item(), near)
    rows, small = [], set()
    for k in ("loss", "loss_sparse", "loss_dense"):
        e, ea = relerr(getattr(out, k), ref[k]), relerr(ac[k], ref[k])
        rows.append((k, e, ea, e, ea))
        small.add(k)
    for name, q in m.named_parameters():
        r = rgrads[name]
        if not bool(r.any()):
            assert q.grad is not None and not bool(q.grad.any()), name
            continue
        rows.append((name + ".grad", frob_relerr(q.grad, r), frob_relerr(agrads[name], r), relerr(q.grad, r), relerr(agrads[name], r)))
        if r.numel() <= 4096:
            small.add(name + ".grad")
    print(f"\n{_cid(case)}: B={B} T={T} L={L}, {B * T} texts, {near} counted positions with a top-1 lead < {cr.MARGIN}, "
          f"fp64 restatement peak {peak:.1f} GiB")
    autocast_yardstick(rows, small)
