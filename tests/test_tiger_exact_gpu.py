"""TIGER's training step under dropout against fp64 references, on the H100.

Part A: every autograd Function of a TIGER block (tiger._RmsNormFn, _LinearFn, _FfnFn, _HeadFn and t5_attention._T5AttnFn in its
five forms) forward and backward on seeded inputs, each stage against its fp64 reference (tests/dense_reference.py,
tests/attention_reference.py) on the kernel's own inputs to that stage.  The forward intermediates come from grad_fn.saved_tensors /
grad_fn.cfg, the backward's from a spy on genrec_b200.functional (cast_rows_bf16, linear_bwd, linear_dact_bwd) and on the attention
core backward.  dy is small integers / 64, so the masked bf16 casts of the backward are exact and checked bit for bit; the dropout
masks are restated from (seed, site), so a backward that pairs a stage with another stage's mask fails here.

Part B: Tiger.forward and forward_jagged, forward and backward, at p = 0.1 and 0.3, against tests/tiger_reference.py in fp64 on the
same masks: torch's F.dropout masks recorded by a shim, the kernels' restated from the step's seed and sites.  The yardstick is the
same restatement under bf16 torch.autocast (exact_check.autocast_yardstick).

`pytest -s` prints the worst error / allowance of every part A quantity and the yardstick table of every part B step."""
import zlib

import pytest
import torch

from tests import attention_reference as ar
from tests import dense_reference as dr
from tests import hstu_block_reference as hr
from tests import tiger_params as tp
from tests import tiger_reference as tr
from tests.exact_check import (FTZ, Ledger, Spy, _TorchDropout, _cid, _dy, _packed_core_ref, _seeded,
                                autocast_yardstick)
from tests.tiger_params import _geometric_lengths, _model, _padded_and_packed

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
WIDTHS = [(64, 2), (128, 4), (384, 6)]
ROWS = [1, 63, 64, 65, 129, 256 * 61]
PS = [0.0, 0.1, 0.3]
LEDGER = Ledger("worst error / allowance per quantity of the TIGER block stages (dense tolerance 1, attention core: "
                "attention_reference.TOL):", width=18, floor=FTZ)
_error_table = LEDGER.fixture()
_check = LEDGER.check


def _spy(monkeypatch):
    """the functional calls of one backward"""
    from genrec_b200 import functional as Fn
    from genrec_b200 import t5_attention as t5
    return Spy(monkeypatch, {Fn: ("cast_rows_bf16", "linear_bwd", "linear_dact_bwd"),
                             t5: ("attention_core_bwd", "attention_core_bwd_jagged")})


# ------------------------------------------------------------------------------------------------ part A: the stages
DENSE_CASES = [(D, H, R, PS[(i + j) % 3]) for i, (D, H) in enumerate(WIDTHS) for j, R in enumerate(ROWS)]


@pytest.mark.parametrize("case", DENSE_CASES, ids=_cid)
def test_rmsnorm_and_linear_stages(case, monkeypatch):
    from genrec_b200.tiger import _LinearFn, _RmsNormFn
    D, H, R, p = case
    x = _seeded((R, D), R + D, 2.0).requires_grad_(True)
    w = (1 + _seeded((D,), 7, 0.1)).requires_grad_(True)
    y = _RmsNormFn.apply(x, w)
    xc, rstd, _ = y.grad_fn.saved_tensors
    dy = _dy((R, D), R)
    spy = _spy(monkeypatch)
    y.backward(dy)
    spy.take()
    fr = dr.rmsnorm_forward(xc, w.detach(), tr.EPS)
    br = dr.rmsnorm_backward(dy, xc, rstd, w.detach())
    items = [("rms y", y.detach(), fr["y"], fr["a_y32"]), ("rms dx", x.grad, br["dx"], br["a_dx"]), ("rms dw", w.grad, br["dw"], br["a_dw"])]
    wl = _seeded((D, D), D, D ** -0.5).requires_grad_(True)
    x.grad = None
    y = _LinearFn.apply(x, wl)
    xb, wb = y.grad_fn.saved_tensors
    assert torch.equal(xb, x.detach().bfloat16()) and torch.equal(wb, wl.detach().bfloat16())
    spy.calls.clear()
    y.backward(dy)
    dyb, (dx, dw, _) = spy.take("cast_rows_bf16", "linear_bwd")
    assert torch.equal(dyb, dr.rne_bf16(dy.double()))
    lf = dr.linear_forward(xb, wb, torch.zeros(D, device=DEV))
    lb = dr.linear_backward(dyb, wb, xb)
    items += [("linear y", y.detach(), lf["z"], lf["a_z"]), ("linear dx", x.grad, lb["dx"], lb["a_dx"]),
              ("linear dw", wl.grad, lb["dw"], lb["a_dw"])]
    _check(_cid(case), items)


@pytest.mark.parametrize("case", DENSE_CASES, ids=_cid)
def test_ffn_stages(case, monkeypatch):
    from genrec_b200.tiger import FFN_DIM, _FfnFn
    D, H, R, p = case
    x = _seeded((R, D), 3 * R + D, 2.0).requires_grad_(True)
    nw = (1 + _seeded((D,), 8, 0.1)).requires_grad_(True)
    wi = _seeded((FFN_DIM, D), D + 1, D ** -0.5).requires_grad_(True)
    wo = _seeded((D, FFN_DIM), D + 2, FFN_DIM ** -0.5).requires_grad_(True)
    torch.manual_seed(R + D)
    y = _FfnFn.apply(x, nw, wi, wo, p)
    xc, rstd, xnb, z, h, wib, wob, _ = y.grad_fn.saved_tensors
    pp, seed, site = y.grad_fn.cfg
    assert pp == p and seed == (torch.initial_seed() & (2 ** 63 - 1) if p > 0 else 0)
    dy = _dy((R, D), R + 1)
    spy = _spy(monkeypatch)
    y.backward(dy)
    dyb, (_, dwo, _), dz, (dxn, dwi, _) = spy.take("cast_rows_bf16", "linear_bwd", "linear_dact_bwd", "linear_bwd")
    zero = torch.zeros(FFN_DIM, device=DEV)
    nf = dr.rmsnorm_forward(xc, nw.detach(), tr.EPS)
    f1 = dr.linear_forward(xnb, wib, zero, 2, z, p, seed, site)
    f2 = dr.linear_residual(h, wob, torch.zeros(D, device=DEV), xc, None, p, seed, site + 1)
    kh = dr.keep(range(R), FFN_DIM, p, seed, site, DEV)
    ko = dr.keep(range(R), D, p, seed, site + 1, DEV)
    # exact: the hidden mask and ReLU in h and dz, the output mask in the cast of dy
    assert torch.equal(h, f1["a_exact"]), "h is not RNE(relu(z) keep(site))"
    dead = (kh == 0) | (z.double() <= 0)
    assert not bool(h[dead].any()) and not bool(dz[dead].any()), "h or dz != 0 where keep(site) drops or z <= 0"
    assert torch.equal(dyb, hr.cast_colsum(dy, p, seed, site + 1)["dyb_exact"]), "dyb is not RNE(keep(site + 1) dy)"
    if p > 0:
        assert bool((kh == 0).any()) and bool((ko == 0).any())
    b2 = dr.linear_backward(dyb, wob, h)
    dzr = hr.linear_dact_backward(dyb, wob, z, p, seed, site, act=2)
    b1 = dr.linear_backward(dz, wib, xnb)
    nb = dr.rmsnorm_backward(dxn, xc, rstd, nw.detach(), res=dy)
    _check(_cid(case), [("ffn xnb", xnb, nf["y"], nf["a_y16"]), ("ffn z", z, f1["z"], f1["a_z"]), ("ffn h", h, f1["a"], f1["a_a"]),
                        ("ffn y", y.detach(), f2["y"], f2["a_y"]), ("ffn dwo", dwo, b2["dw"], b2["a_dw"]),
                        ("ffn dz", dz, dzr["g"], dzr["a_g"]), ("ffn dxn", dxn, b1["dx"], b1["a_dx"]), ("ffn dwi", dwi, b1["dw"], b1["a_dw"]),
                        ("ffn dx", x.grad, nb["dx"], nb["a_dx"]), ("ffn dnw", nw.grad, nb["dw"], nb["a_dw"])])
    assert torch.equal(wi.grad, dwi) and torch.equal(wo.grad, dwo)


@pytest.mark.parametrize("case", [(D, H, R) for (D, H) in WIDTHS for R in (1, 65, 129, 256 * 3)], ids=_cid)
def test_head_stages(case, monkeypatch):
    from genrec_b200.tiger import _HeadFn
    D, H, R = case
    V = 769
    x = _seeded((R, D), R + 5, 2.0).requires_grad_(True)
    w = _seeded((V, D), D + 3, D ** -0.5).requires_grad_(True)
    y = _HeadFn.apply(x, w)
    xb, wp = y.grad_fn.saved_tensors
    assert wp.shape == (776, D) and not bool(wp[V:].any()) and torch.equal(wp[:V], w.detach().bfloat16())
    dy = _dy((R, V), R + 2)
    spy = _spy(monkeypatch)
    y.backward(dy)
    dyb, (dx, dwp, _) = spy.take("cast_rows_bf16", "linear_bwd")
    assert not bool(dyb[:, V:].any()) and not bool(dwp[V:].any()), "a pad row of the head mirror reached dw"
    lf = dr.linear_backward(xb, wp.t().contiguous(), xb)
    lb = dr.linear_backward(dyb, wp, xb)
    _check(_cid(case), [("head logits", y.detach(), lf["dx"][:, :V], lf["a_dx"][:, :V]), ("head dx", x.grad, lb["dx"], lb["a_dx"]),
                        ("head dw", w.grad, lb["dw"][:V], lb["a_dw"][:V])])


# ---- attention: (form, lengths | (B, L), Lq, D, H, p)
ATTN_CASES = [
    ("encoder", (1, 1), 0), ("encoder", (1, 63), 0), ("encoder", (1, 64), 0), ("encoder", (1, 65), 0), ("encoder", (3, 43), 0),
    ("encoder", (256, 61), 0),
    ("decoder", (1, 4), 0), ("decoder", (16, 4), 0), ("decoder", (33, 4), 0), ("decoder", (256, 4), 0),
    ("cross", (1, 1), 4), ("cross", (16, 4), 4), ("cross", (5, 65), 4), ("cross", (256, 61), 4),
    ("packed self", [1, 31, 61, 64, 67], 0), ("packed self", [1], 0), ("packed self", [63, 1, 65], 0), ("packed self", "geometric", 0),
    ("packed cross", [1, 31, 61, 64, 67], 4), ("packed cross", [65, 1], 4), ("packed cross", "geometric", 4),
]
ATTN = [(f, shp, Lq, D, H, PS[(i + j) % 3]) for i, (f, shp, Lq) in enumerate(ATTN_CASES) for j, (D, H) in enumerate(WIDTHS)]


def _lengths(shp):
    if shp == "geometric":                             # the published step's memories: 1 + 3 items each
        return [1 + 3 * n for n in _geometric_lengths(256, 4)]
    return list(shp)


def _aid(c):
    f, shp, Lq, D, H, p = c
    return f"{f}-{shp if isinstance(shp, str) else 'x'.join(map(str, shp))}-D{D}-H{H}-p{p}"


@pytest.mark.parametrize("case", ATTN, ids=_aid)
def test_t5_attention_stages(case, monkeypatch):
    from genrec_b200 import t5_attention as t5
    from genrec_b200.t5_attention import _T5AttnFn
    form, shp, Lq, D, H, p = case
    packed = form.startswith("packed")
    cross = form.endswith("cross")
    causal = form == "decoder"
    seed_in = D + H + zlib.crc32(str(shp).encode())
    idle = 0
    if packed:
        lengths = _lengths(shp)
        idle = 3 if form == "packed self" else 0
        offs = [0]
        for n in lengths:
            offs.append(offs[-1] + n)
        T, B, mx = offs[-1] + idle, len(lengths), max(lengths)
        offsets = torch.tensor(offs, dtype=torch.int64, device=DEV)
        jag = (offsets, mx)
    else:
        B, L = shp
        jag = ()
    if form in ("encoder", "decoder"):
        xq, xm, Lk = _seeded((B, L, D), seed_in, 2.0), None, L
    elif form == "cross":
        xq, xm, Lk = _seeded((B, Lq, D), seed_in, 2.0), _seeded((B, L, D), seed_in + 1, 2.0), L
    elif form == "packed self":
        xq, xm, Lk = _seeded((T, D), seed_in, 2.0), None, mx
    else:
        xq, xm, Lk = _seeded((B, Lq, D), seed_in, 2.0), _seeded((T, D), seed_in + 1, 2.0), mx
    query = xq.requires_grad_(True)
    mem = xm.requires_grad_(True) if xm is not None else None
    wq = _seeded((D, D), 1, D ** -0.5).requires_grad_(True)
    wo = _seeded((D, D), 2, D ** -0.5).requires_grad_(True)
    if cross:
        wk, wv, rel = _seeded((D, D), 3, D ** -0.5).requires_grad_(True), _seeded((D, D), 4, D ** -0.5).requires_grad_(True), None
        bucket = None
    else:
        wk, wv = _seeded((2 * D, D), 5, D ** -0.5).requires_grad_(True), None
        rel = _seeded((H * 32, 1), 6, 0.5).requires_grad_(True)
        bucket = t5._bucket_map(Lk, Lk, 32, 128, DEV)
    key_pad = None
    if form in ("encoder", "cross") and B > 1:
        n_valid = torch.arange(B) * 7 % Lk + 1                # every sequence keeps its first key (the user row)
        key_pad = (torch.arange(Lk)[None, :] >= n_valid[:, None]).to(torch.uint8).to(DEV)
    torch.manual_seed(D * 31 + B)
    out = _T5AttnFn.apply(query, mem, mem, key_pad, causal, H, p, bucket, wq, wk, wv, wo, rel, not cross, *jag)
    sv = out.grad_fn.saved_tensors
    xqb, xkb, _, Q, K, V, A, _, wqb, wkb, wvb, wob, bias = sv[:13]
    Hc, pc, seed, site, scale, *_ = out.grad_fn.cfg
    assert (Hc, pc) == (H, p) and seed == (torch.initial_seed() & (2 ** 63 - 1) if p > 0 else 0) and site == t5._CALLS["n"]
    bias = bias if rel is not None else None
    dy = _dy(tuple(out.shape), D + B)
    spy = _spy(monkeypatch)
    out.backward(dy)
    core = "attention_core_bwd_jagged" if packed else "attention_core_bwd"
    if cross:
        dyb, (dA, dwo, _), dAb, (dQ, dK32, dV32, dbias), (dq_x, dwq, _), dKb, (dk_x, dwk, _), dVb, (dv_x, dwv, _) = spy.take(
            "cast_rows_bf16", "linear_bwd", "cast_rows_bf16", core, "linear_bwd", "cast_rows_bf16", "linear_bwd", "cast_rows_bf16",
            "linear_bwd")
    else:
        dyb, (dA, dwo, _), dAb, (dQ, dK32, dV32, dbias), dKV, (dx_kv, dwkv, _), (dq_x, dwq, _) = spy.take(
            "cast_rows_bf16", "linear_bwd", "cast_rows_bf16", core, "cast_rows_bf16", "linear_bwd", "linear_bwd")
    case_id = _aid(case)
    flat = lambda t: t.reshape(-1, t.shape[-1])
    zD = torch.zeros(D, device=DEV)
    # projections
    pq = dr.linear_forward(flat(xqb), wqb, zD)
    items = [("attn Q", flat(Q), pq["z"], pq["a_z"])]
    if cross:
        pk, pv = dr.linear_forward(flat(xkb), wkb, zD), dr.linear_forward(flat(xkb), wvb, zD)
        items += [("attn K", flat(K), pk["z"], pk["a_z"]), ("attn V", flat(V), pv["z"], pv["a_z"])]
    else:
        pkv = dr.linear_forward(flat(xqb), wkb, torch.zeros(2 * D, device=DEV))
        items += [("attn K|V", torch.cat([flat(K), flat(V)], -1), pkv["z"], pkv["a_z"])]
    po = dr.linear_forward(flat(A), wob, zD)
    items.append(("attn out", out.detach().reshape(-1, D), po["z"], po["a_z"]))
    # the core on its own inputs
    assert torch.equal(dyb, dr.rne_bf16(dy.double())) and torch.equal(dAb, dA.bfloat16())
    if packed:
        ref = _packed_core_ref(Q, K, V, A, dAb, H, bias, offs, Lq, scale, p, seed, site)
        seq_q = slice(0, offs[-1]) if Lq == 0 else slice(None)
        got = {"out": A[seq_q].reshape(-1, D), "dq": dQ[seq_q].reshape(-1, D), "dk": dK32[:offs[-1]], "dv": dV32[:offs[-1]]}
        if Lq == 0:
            assert not bool(A[offs[-1]:].any()) and not bool(dQ[offs[-1]:].any()), "an idle row has an attention output or dQ"
        assert not bool(dK32[offs[-1]:].any()) and not bool(dV32[offs[-1]:].any()), "an idle row has dK or dV"
    else:
        ref = ar.t5_reference(Q, K, V, H, bias, bucket, key_pad, causal, scale, dAb, A, p, seed, site)
        got = {"out": A, "dq": dQ, "dk": dK32, "dv": dV32}
        assert not ar.t5_exact(got, ref, key_pad)
        if p > 0 and ref["drop"].numel() >= 64:
            assert bool(ref["drop"].any())
    if bias is not None:
        got["dbias"] = dbias
    LEDGER.check_core(case_id, ar.errors(got, ref, ("out", "dq", "dk", "dv", "dbias")), "t5")
    # backward projections
    bo = dr.linear_backward(flat(dyb), wob, flat(A))
    items += [("attn dA", flat(dA), bo["dx"], bo["a_dx"]), ("attn dwo", dwo, bo["dw"], bo["a_dw"])]
    if cross:
        assert torch.equal(dKb, dK32.bfloat16()) and torch.equal(dVb, dV32.bfloat16())
        bq = dr.linear_backward(flat(dQ), wqb, flat(xqb))
        bk, bv = dr.linear_backward(flat(dKb), wkb, flat(xkb)), dr.linear_backward(flat(dVb), wvb, flat(xkb))
        items += [("attn dwq", dwq, bq["dw"], bq["a_dw"]), ("attn dwk", dwk, bk["dw"], bk["a_dw"]), ("attn dwv", dwv, bv["dw"], bv["a_dw"]),
                  ("attn dquery", query.grad.reshape(-1, D), bq["dx"], bq["a_dx"]),
                  ("attn dkey+dvalue", mem.grad.reshape(-1, D), bk["dx"] + bv["dx"], bk["a_dx"] + bv["a_dx"] + dr.C * (bk["dx"] + bv["dx"]).abs())]
        assert torch.equal(wk.grad, dwk) and torch.equal(wv.grad, dwv)
    else:
        assert torch.equal(dKV, torch.cat([dK32, dV32], -1).bfloat16())
        bkv = dr.linear_backward(flat(dKV), wkb, flat(xqb))
        bq = dr.linear_backward(flat(dQ), wqb, flat(xqb), res=dx_kv.reshape(-1, D))
        items += [("attn dx_kv", flat(dx_kv), bkv["dx"], bkv["a_dx"]), ("attn dwkv", dwkv, bkv["dw"], bkv["a_dw"]),
                  ("attn dwq", dwq, bq["dw"], bq["a_dw"]), ("attn dquery", query.grad.reshape(-1, D), bq["dx"], bq["a_dx"])]
        assert torch.equal(rel.grad.view(H, -1), dbias) and torch.equal(wk.grad, dwkv)
    assert torch.equal(wq.grad, dwq) and torch.equal(wo.grad, dwo)
    _check(case_id, items)


def test_edges_are_reached():
    """rows at and around the 64-row GEMM and core tiles and the published step; the core at dh 32 and 64; every p"""
    assert {1, 63, 64, 65, 129, 15616} <= {c[2] for c in DENSE_CASES}
    assert {(D // H) for D, H, _, _ in DENSE_CASES} == {32, 64}
    assert {(c[2], c[3]) for c in DENSE_CASES} >= {(15616, 0.0), (15616, 0.1)} and {c[3] for c in DENSE_CASES} == set(PS)
    forms = {c[0] for c in ATTN}
    assert forms == {"encoder", "decoder", "cross", "packed self", "packed cross"}
    for f in forms:
        assert {c[5] for c in ATTN if c[0] == f} == set(PS), f
    mem = {n for c in ATTN if c[0].startswith("packed") for n in _lengths(c[1])}
    assert {1, 31, 61, 64, 67} <= mem
    assert {c[1][1] for c in ATTN if c[0] == "encoder"} >= {1, 63, 64, 65}


# ------------------------------------------------------------------------------------------------ part B: the whole step


def _graph_cfgs(root):
    """cfg of every _T5AttnFn / _FfnFn node reachable from root"""
    seen, todo, cfgs = set(), [root], {"attn": [], "ffn": []}
    while todo:
        f = todo.pop()
        if f is None or f in seen:
            continue
        seen.add(f)
        name = type(f).__name__
        if "T5AttnFn" in name:
            cfgs["attn"].append(f.cfg)
        elif "FfnFn" in name:
            cfgs["ffn"].append(f.cfg)
        todo.extend(n for n, _ in f.next_functions)
    return cfgs


STEPS = [(shape, p, form) for shape in ("small", "published") for p in (0.1, 0.3) for form in ("padded", "packed")]
STEPS += [("edges", p, form) for p in (0.1, 0.3) for form in ("padded", "packed", "packed idle")]


@pytest.mark.parametrize("case", STEPS, ids=_cid)
def test_training_step_vs_fp64(case, monkeypatch):
    from genrec_b200 import t5_attention, tiger
    from tests.util import frob_relerr, relerr
    shape, p, form = case
    # B = 256 throughout: the yardstick compares two realisations of bf16 noise, which a handful of users leaves too scattered
    if shape == "edges":                               # memories of 1, 31, 61, 64 and 67 rows: the core's tile edges
        cfg, B, n, lengths = dict(tp.PUBLISHED), 255, 22, [0, 10, 20, 21, 22] * 51
    else:
        cfg, B, n = dict(tp.PUBLISHED if shape == "published" else tp.SMALL), 256, (20 if shape == "published" else 6)
        lengths = _geometric_lengths(B, 1, cap=n)
    cfg["dropout"] = p
    padded, pk = _padded_and_packed(cfg, B, n, 3, lengths)
    if form == "packed idle":
        T = int(pk["mem_offsets"][-1]) + 37
        _, pk = _padded_and_packed(cfg, B, n, 3, lengths, num_tokens=T)
        assert pk["item_input_ids"].numel() == T and pk["max_len"] == 1 + 3 * n and not bool(pk["overflow"])
    if shape == "edges":
        assert (pk["mem_offsets"][1:] - pk["mem_offsets"][:-1]).tolist() == [1, 31, 61, 64, 67] * 51
    m = _model(cfg).train()
    shim = _TorchDropout()
    monkeypatch.setattr(tiger, "F", shim)
    torch.manual_seed(1000 + B + int(10 * p))
    seed = torch.initial_seed() & (2 ** 63 - 1)
    a0, f0 = t5_attention._CALLS["n"], tiger._SITES["n"]
    if form == "padded":
        out = m(padded["user_input_ids"], padded["item_input_ids"], padded["token_type_ids"], padded["target_input_ids"],
                padded["target_token_type_ids"], padded["seq_mask"])
        batch, mem = padded, ("padded", padded["item_input_ids"].shape[1] + 1)
    else:
        out = m.forward_jagged(pk["user_input_ids"], pk["item_input_ids"], pk["token_type_ids"], pk["mem_offsets"], pk["max_len"],
                               pk["target_input_ids"], pk["target_token_type_ids"])
        batch, mem = {k: v for k, v in pk.items() if k != "overflow"}, ("packed", pk["item_input_ids"].numel(), pk["max_len"])
    out.loss.backward()
    S1 = out.logits.shape[1]
    masks = tr.kernel_step_masks(cfg, shim.masks, p, seed, a0, f0, B, S1, mem, DEV)
    # the restated sites and seeds are those of the graph's Functions
    cfgs = _graph_cfgs(out.loss.grad_fn)
    n_blk = cfg["n_layers"] // 2
    assert sorted(c[3] for c in cfgs["attn"]) == list(range(a0 + 1, a0 + 3 * n_blk + 1))
    assert sorted(c[2] for c in cfgs["ffn"]) == list(range(f0 + 2, f0 + 4 * n_blk + 1, 2))
    assert {c[2] for c in cfgs["attn"]} == {seed} and {c[1] for c in cfgs["ffn"]} == {seed}
    assert t5_attention._CALLS["n"] == a0 + 3 * n_blk and tiger._SITES["n"] == f0 + 4 * n_blk
    for i, k in enumerate(masks):                      # every source drops something
        assert bool((k == 0).any()), f"mask {i} {tuple(k.shape)} keeps everything"
    params = {k: v.detach() for k, v in m.state_dict().items()}
    packed = form != "padded"
    ref = tr.step(params, cfg, batch, masks, packed, device=DEV)
    ac = tr.step(params, cfg, batch, masks, packed, dtype=torch.float32, device=DEV, autocast=True)
    el, ea = abs(out.loss.item() - ref["loss"].item()) / abs(ref["loss"].item()), abs(ac["loss"].item() - ref["loss"].item()) / abs(ref["loss"].item())
    rows = [("loss", el, ea, el, ea),
            ("logits", frob_relerr(out.logits, ref["logits"]), frob_relerr(ac["logits"], ref["logits"]), relerr(out.logits, ref["logits"]),
             relerr(ac["logits"], ref["logits"]))]
    small = set()
    for name, q in m.named_parameters():
        if name not in ref["grads"]:
            assert q.grad is None or not bool(q.grad.any()), name
            continue
        g, r = q.grad, ref["grads"][name]
        if r.abs().max() == 0:
            assert g.abs().max() == 0, name
            continue
        rows.append((name + ".grad", frob_relerr(g, r), frob_relerr(ac["grads"][name], r), relerr(g, r), relerr(ac["grads"][name], r)))
        if r.numel() <= 4096:                           # SMALL's 64 x 64 matrices scatter like the small vectors
            small.add(name + ".grad")
    print(f"\n{_cid(case)}")
    autocast_yardstick(rows, small)
