"""SASRec's training step under dropout against fp64 references, on the H100.

Part A: every stage of sasrec._BlockFn forward and backward, each against its fp64 reference (tests/dense_reference.py,
tests/attention_reference.py, tests/hstu_block_reference.py) on the kernel's own inputs to that stage.  The forward intermediates
come from grad_fn.saved_tensors / grad_fn.cfg and a spy on layernorm_fwd (the fp32 LN1 output qf, which is not saved), the
backward's from a spy on genrec_b200.functional (cast_rows_bf16, linear_bwd, linear_dact_bwd, layernorm_bwd, sasrec_attention_bwd;
the spy also sees the calls ffn_bwd makes).  dy is small integers / 64, so the masked bf16 casts of the backward are exact and
checked bit for bit; the dropout masks are restated from (seed, seed_dev, site, row key), so a stage paired with another stage's
mask, a residual taken from the wrong tensor or a packed batch keyed like a padded one fails here.

Part B: SASRec.forward and forward_jagged, loss and backward, at p = 0.2 and 0.5, against tests/sasrec_reference.py in fp64 on the
masks the kernels draw (sasrec_reference.kernel_step_masks).  The yardstick is the same restatement under bf16 torch.autocast
(exact_check.autocast_yardstick).

Part C: the stand-alone layers (MultiHeadAttention, PointWiseFeedForward, SASRecBlock, HSTULayer) in training at p = 0.5 draw a
fresh mask on every call, each call computes what its own seeds restate, and a backward re-derives its forward's masks even after
another forward has run.

`pytest -s` prints the worst error / allowance of every part A quantity and the yardstick table of every part B step."""
import pytest
import torch

from tests import attention_reference as ar
from tests import dense_reference as dr
from tests import hstu_block_reference as hr
from tests import sasrec_reference as sr
from tests.exact_check import FTZ, Ledger, Spy, _cid, _dy, _seeded, autocast_yardstick

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
LEDGER = Ledger("worst error / allowance per quantity of the SASRec block stages (dense tolerance 1, attention core: "
                "attention_reference.TOL['sas *']):", width=14, floor=FTZ)
_error_table = LEDGER.fixture()
_check = LEDGER.check
SEED, SEED_DEV = 0x1234_5678_9ABC_DEF, 0x9E3779B1 * 3


def _fwd_spy(monkeypatch):
    from genrec_b200 import functional as Fn
    return Spy(monkeypatch, {Fn: ("layernorm_fwd",)})


def _bwd_spy(monkeypatch):
    from genrec_b200 import functional as Fn
    return Spy(monkeypatch, {Fn: ("cast_rows_bf16", "linear_bwd", "linear_dact_bwd", "layernorm_bwd", "sasrec_attention_bwd")})


def _block(D, H, p, layer, seed):
    """a training SASRecBlock with seeded weights, norm gains and biases (none at 1 or 0)"""
    from genrec_b200.sasrec import SASRecBlock
    blk = SASRecBlock(D, H, 4 * D, p)
    prm = sr.seeded_params(dict(num_items=1, max_seq_len=1, embed_dim=D, ffn_dim=4 * D, num_blocks=1), seed)
    blk.load_state_dict({k[len("blocks.0."):]: v for k, v in prm.items() if k.startswith("blocks.0.")})
    blk.layer_index = layer
    return blk.to(DEV).train()


def _core_ref(Q, K, V, pad, H, datt, att, p, seed, layer, offsets):
    """the fp64 attention core on the kernel's bf16 Q, K, V, dO and O: one padded batch, or sequence by sequence with the packed
    row keys (the rows of every sequence, in order)"""
    if offsets is None:
        return ar.sasrec_reference(Q, K, V, pad, H, datt, att, p, seed, layer)
    names = ("out", "dq", "dk", "dv")
    cat = {k: [] for n in names for k in (n, "a_" + n)}
    qpad, saved = [], ar.attn_keep
    try:
        for a, b in zip(offsets, offsets[1:]):
            if b == a:
                continue
            ar.attn_keep = lambda B, H_, Lq, Lk, p_, s_, site, device="cpu", a=a: sr.packed_attn_keep(a, Lq, H_, p_, s_, site, device)
            s = slice(a, b)
            r = ar.sasrec_reference(Q[s][None], K[s][None], V[s][None], pad[s][None], H, datt[s][None], att[s][None], p, seed, layer)
            for k in cat:
                cat[k].append(r[k][0])
            qpad.append(r["qpad"][0])
    finally:
        ar.attn_keep = saved
    ref = {k: torch.cat(v) for k, v in cat.items()}
    ref["qpad"] = torch.cat(qpad)
    return ref


def _forward_items(case_id, y, qf, blk, offsets, eff):
    """every forward stage of one _BlockFn call on its own inputs; returns what the backward checks reuse"""
    x, rowmask, pad, st1, st2, qb, xb, Q, K, V, att, lse, h, hnb, z1, a1, g1, g2 = y.grad_fn.saved_tensors
    cfg, w = y.grad_fn.cfg, y.grad_fn.bf16w
    p, layer, H = cfg["p"], cfg["layer"], cfg["H"]
    fl = lambda t: t.reshape(-1, t.shape[-1])
    xf, z1, a1, st1, st2 = fl(x), fl(z1), fl(a1), fl(st1), fl(st2)
    T, D = xf.shape
    a, f = blk.attention, blk.ffn
    ln1 = dr.layernorm_forward(xf, g1, blk.norm1.bias.detach(), sr.EPS)
    assert torch.equal(xb, x.bfloat16()), "xb is not RNE(x)"
    items = [("ln1 qb", fl(qb), ln1["y"], ln1["a_y16"]), ("ln1 qf", fl(qf), ln1["y"], ln1["a_y32"]),
             ("ln1 mean", st1[:, 0], ln1["mean"], ln1["a_mean"]), ("ln1 rstd", st1[:, 1], ln1["rstd"], ln1["a_rstd"])]
    pq = dr.linear_forward(fl(qb), w["wq"], a.q_proj.bias.detach())
    pk = dr.linear_forward(fl(xb), w["wk"], a.k_proj.bias.detach())
    pv = dr.linear_forward(fl(xb), w["wv"], a.v_proj.bias.detach())
    items += [("Q", fl(Q), pq["z"], pq["a_z"]), ("K", fl(K), pk["z"], pk["a_z"]), ("V", fl(V), pv["z"], pv["a_z"])]
    href = fl(att).double() + fl(qf).double()
    items.append(("h", fl(h), href, dr.C * href.abs()))
    ln2 = dr.layernorm_forward(fl(h), g2, blk.norm2.bias.detach(), sr.EPS)
    items += [("ln2 hnb", fl(hnb), ln2["y"], ln2["a_y16"]), ("ln2 mean", st2[:, 0], ln2["mean"], ln2["a_mean"]),
              ("ln2 rstd", st2[:, 1], ln2["rstd"], ln2["a_rstd"])]
    f1 = dr.linear_forward(fl(hnb), w["w1"], f.fc1.bias.detach(), 2, z1, p, eff, hr.site(layer, sr.SITE_HID))
    assert torch.equal(a1, f1["a_exact"]), "a1 is not RNE(relu(z1) keep(8 layer + 1))"
    rs = rowmask if cfg["apply_mask"] else None
    f2 = dr.linear_residual(a1, w["w2"], f.fc2.bias.detach(), fl(h), rs, p, eff, hr.site(layer, sr.SITE_OUT))
    items += [("ffn z1", z1, f1["z"], f1["a_z"]), ("ffn a1", a1, f1["a"], f1["a_a"]), ("y", fl(y.detach()), f2["y"], f2["a_y"])]
    if p > 0 and T >= 64:
        assert bool((f1["a"][f1["z"] > 0] == 0).any()), "the hidden dropout drops nothing"
    _check(case_id, items)
    return dict(x=xf, rowmask=rowmask, pad=pad, st1=st1, st2=st2, qb=fl(qb), xb=fl(xb), Q=Q, K=K, V=V, att=att, h=fl(h), hnb=fl(hnb),
                z1=z1, a1=a1, g1=g1, g2=g2, w=w, cfg=cfg, D=D, offsets=offsets)


def _backward_items(case_id, blk, s, dy, spy, x_grad, eff):
    """every backward stage of one _BlockFn call on its own inputs, from the spy's record of that backward"""
    (dyb, (none, dw2, db2), dz1, (dhn, dw1, db1), (dh, dg2, dbt2), datt, (dQ, dK, dV), (dq, dwq, dbq), (dxk, dwk, dbk),
     (dxkv, dwv, dbv), (dx, dg1, dbt1)) = spy.take("cast_rows_bf16", "linear_bwd", "linear_dact_bwd", "linear_bwd", "layernorm_bwd",
                                                   "cast_rows_bf16", "sasrec_attention_bwd", "linear_bwd", "linear_bwd", "linear_bwd",
                                                   "layernorm_bwd")
    assert none is None
    cfg, w, layer, p, H = s["cfg"], s["w"], s["cfg"]["layer"], s["cfg"]["p"], s["cfg"]["H"]
    fl = lambda t: t.reshape(-1, t.shape[-1])
    dym = fl(dy) * s["rowmask"][:, None] if cfg["apply_mask"] else fl(dy)
    cc = hr.cast_colsum(dym, p, eff, hr.site(layer, sr.SITE_OUT))
    assert torch.equal(fl(dyb), cc["dyb_exact"]), "dyb is not RNE(keep(8 layer + 2) dy rowmask)"
    b2 = dr.linear_backward(fl(dyb), w["w2"], s["a1"])
    dzr = hr.linear_dact_backward(fl(dyb), w["w2"], s["z1"], p, eff, hr.site(layer, sr.SITE_HID), act=2)
    dz1 = fl(dz1)
    b1 = dr.linear_backward(dz1, w["w1"], s["hnb"])
    n2 = dr.layernorm_backward(fl(dhn), s["h"], s["st2"], s["g2"], res=dym)
    assert torch.equal(fl(datt), fl(dh).bfloat16()), "datt is not RNE(dh)"
    ref = _core_ref(s["Q"], s["K"], s["V"], s["pad"], H, datt, s["att"], p, eff, layer, s["offsets"])
    got = {"out": s["att"], "dq": dQ, "dk": dK, "dv": dV}
    if s["offsets"] is not None:                       # the core's rows: the sequences'; the idle rows after them are exact zeros
        n = s["offsets"][-1]
        for k, t in got.items():
            assert not bool(t[n:].any()), f"an idle row has {k} != 0"
        got = {k: t[:n] for k, t in got.items()}
    LEDGER.check_core(case_id, ar.errors(got, ref, ("out", "dq", "dk", "dv")), "sas")
    assert not ar.sasrec_exact(got, ref)
    if p > 0 and ref["out"].numel() >= 4096 and s["offsets"] is None:
        assert bool(ref["drop"][ref["valid"]].any()), "the attention dropout drops nothing"
    bq = dr.linear_backward(fl(dQ), w["wq"], s["qb"], res=fl(dh))
    bk = dr.linear_backward(fl(dK), w["wk"], s["xb"])
    bv = dr.linear_backward(fl(dV), w["wv"], s["xb"], res=fl(dxk))
    n1 = dr.layernorm_backward(fl(dq), s["x"], s["st1"], s["g1"], res=fl(dxkv))
    items = [("dw2", dw2, b2["dw"], b2["a_dw"]), ("db2", db2, b2["db"], b2["a_db"]), ("dz1", dz1, dzr["g"], dzr["a_g"]),
             ("dhn", fl(dhn), b1["dx"], b1["a_dx"]), ("dw1", dw1, b1["dw"], b1["a_dw"]), ("db1", db1, b1["db"], b1["a_db"]),
             ("dh", fl(dh), n2["dx"], n2["a_dx"]), ("dg2", dg2, n2["dg"], n2["a_dg"]), ("dbt2", dbt2, n2["db"], n2["a_db"]),
             ("dq", fl(dq), bq["dx"], bq["a_dx"]), ("dwq", dwq, bq["dw"], bq["a_dw"]), ("dbq", dbq, bq["db"], bq["a_db"]),
             ("dxk", fl(dxk), bk["dx"], bk["a_dx"]), ("dwk", dwk, bk["dw"], bk["a_dw"]), ("dbk", dbk, bk["db"], bk["a_db"]),
             ("dxkv", fl(dxkv), bv["dx"], bv["a_dx"]), ("dwv", dwv, bv["dw"], bv["a_dw"]), ("dbv", dbv, bv["db"], bv["a_db"]),
             ("dx", fl(dx), n1["dx"], n1["a_dx"]), ("dg1", dg1, n1["dg"], n1["a_dg"]), ("dbt1", dbt1, n1["db"], n1["a_db"])]
    _check(case_id, items)
    assert torch.equal(x_grad.reshape(-1, s["D"]), fl(dx))
    a, f = blk.attention, blk.ffn
    for prm, g in ((blk.norm1.weight, dg1), (blk.norm1.bias, dbt1), (a.q_proj.weight, dwq), (a.q_proj.bias, dbq), (a.k_proj.weight, dwk),
                   (a.k_proj.bias, dbk), (a.v_proj.weight, dwv), (a.v_proj.bias, dbv), (blk.norm2.weight, dg2), (blk.norm2.bias, dbt2),
                   (f.fc1.weight, dw1), (f.fc1.bias, db1), (f.fc2.weight, dw2), (f.fc2.bias, db2)):
        assert torch.equal(prm.grad, g)
    if p > 0:
        assert bool(cc["drop"].any()), "the FFN output dropout drops nothing"


# ------------------------------------------------------------------------------------------------ part A: the stages
LS = [1, 50, 63, 64, 65, 129, 200]
PS = [0.0, 0.2, 0.5]
LAYERS = [0, 1, 3]
# (B, L, dh, H, p, layer, with a device seed)
PADDED = [(5, L, dh, 2, PS[(i + j) % 3], LAYERS[(i + 2 * j) % 3], (i + j) % 2 == 1) for i, L in enumerate(LS) for j, dh in enumerate((32, 64))]
PADDED += [(128, 50, 32, 2, 0.2, 1, True), (128, 50, 32, 2, 0.5, 0, False)]      # the reference block: B = 128, L = 50, d = 64
PACK_LENGTHS = [0, 1, 63, 64, 65, 127, 128, 129, 200]
PACKED = [(dh, p, layer, sd) for dh, p, layer, sd in ((32, 0.2, 1, True), (64, 0.5, 3, False), (64, 0.0, 0, False), (32, 0.5, 0, True))]


def _padded_inputs(B, L, D, seed):
    """x ~ N(0, 1) zeroed at the pads (as the model feeds a block); pads: left (row 0), a hole mid-sequence (row 1), every position
    (row 2); a row of exact zeros and a constant row among the real tokens of row 3 (LayerNorm's variance is 0 there: rstd = 1e4)"""
    x = _seeded((B, L, D), seed)
    mask = torch.ones(B, L, device=DEV)
    if B >= 4:
        mask[0, : (L + 1) // 3] = 0
        mask[1, L // 2: L // 2 + max(1, L // 5)] = 0 if L > 2 else 1
        mask[2] = 0
        x[3, L // 2] = 0
        x[3, (L - 1) // 3] = 0.1
    if B > 8:
        mask[8:, : L // 4] = 0                           # the reference block: left-padded users
    return x * mask[..., None], mask


def _block_case(case_id, blk, run, x, dy, monkeypatch, eff, offsets):
    xg = x.clone().requires_grad_(True)
    fs = _fwd_spy(monkeypatch)
    y = run(xg)
    (_, qf, _), _ = fs.take("layernorm_fwd", "layernorm_fwd")
    s = _forward_items(case_id, y, qf, blk, offsets, eff)
    bs = _bwd_spy(monkeypatch)
    y.backward(dy)
    _backward_items(case_id, blk, s, dy, bs, xg.grad, eff)
    return y


@pytest.mark.parametrize("case", PADDED, ids=_cid)
def test_block_stages_padded(case, monkeypatch):
    B, L, dh, H, p, layer, with_sd = case
    D = H * dh
    blk = _block(D, H, p, layer, L + dh)
    x, mask = _padded_inputs(B, L, D, 3 * L + dh)
    sd = torch.tensor([SEED_DEV], dtype=torch.int64, device=DEV) if with_sd else None
    eff = hr.effective_seed(SEED, p, SEED_DEV if with_sd else None)
    dy = _dy((B, L, D), L + B)
    y = _block_case(_cid(case), blk, lambda xg: blk(xg, mask[..., None], _apply_mask=True, _seed=SEED, _seed_dev=sd), x, dy, monkeypatch,
                    eff, None)
    cfg = y.grad_fn.cfg
    assert (cfg["layer"], cfg["p"], cfg["seed"], cfg["seed_dev"] is sd) == (layer, p, SEED, True)


@pytest.mark.parametrize("case", PACKED, ids=_cid)
def test_block_stages_packed(case, monkeypatch):
    """a packed batch over sequences of 0, 1, 63, 64, 65, 127, 128, 129 and 200 rows, an id-0 token in two of them and 37 idle
    rows after them: the core keys its dropout by token row (tok0 + i) H + h"""
    dh, p, layer, with_sd = case
    H = 2
    D = H * dh
    offs = [0]
    for n in PACK_LENGTHS:
        offs.append(offs[-1] + n)
    T = offs[-1] + 37
    blk = _block(D, H, p, layer, 7 + dh)
    rowmask = torch.zeros(T, device=DEV)
    rowmask[:offs[-1]] = 1
    rowmask[[offs[3] + 5, offs[8] + 100]] = 0
    pad = (rowmask == 0).to(torch.uint8)
    x = _seeded((T, D), 11 + dh) * rowmask[:, None]
    sd = torch.tensor([SEED_DEV], dtype=torch.int64, device=DEV) if with_sd else None
    eff = hr.effective_seed(SEED, p, SEED_DEV if with_sd else None)
    offsets = torch.tensor(offs, dtype=torch.int64, device=DEV)
    dy = _dy((T, D), T)
    _block_case(_cid(case), blk, lambda xg: blk._run(xg, rowmask, pad, True, SEED, sd, offsets, 200), x, dy, monkeypatch, eff, offs)


def test_edges_are_reached():
    """rows at and around the 64-row core tiles and past 128; head dim 32 and 64; every p at each head dim; layers 0, 1 and 3; the
    device seed on and off; the reference block; a packed batch at the same edges"""
    assert {c[1] for c in PADDED} >= {1, 50, 63, 64, 65, 129, 200}
    for dh in (32, 64):
        assert {c[4] for c in PADDED if c[2] == dh} == set(PS), dh
    assert {c[5] for c in PADDED} == set(LAYERS) and {c[6] for c in PADDED} == {True, False}
    assert (128, 50, 32, 2) in {c[:4] for c in PADDED}
    assert {1, 63, 64, 65, 127, 128, 129, 200} <= set(PACK_LENGTHS) and 0 in PACK_LENGTHS
    assert {c[0] for c in PACKED} == {32, 64} and {c[1] for c in PACKED} == set(PS) and {c[3] for c in PACKED} == {True, False}


# ------------------------------------------------------------------------------------------------ part B: the whole step
def _block_cfgs(root):
    """cfg of every _BlockFn node reachable from root"""
    seen, todo, cfgs = set(), [root], []
    while todo:
        f = todo.pop()
        if f is None or f in seen:
            continue
        seen.add(f)
        if "_BlockFn" in type(f).__name__:
            cfgs.append(f.cfg)
        todo.extend(n for n, _ in f.next_functions)
    return cfgs


REFERENCE = dict(num_items=12101, max_seq_len=50, embed_dim=64, num_heads=2, num_blocks=2, ffn_dim=256)
EDGE = [dict(num_items=12101, max_seq_len=200, embed_dim=128, num_heads=H, num_blocks=2, ffn_dim=512) for H in (4, 2)]
STEPS = [("reference", p, form) for p in (0.2, 0.5) for form in ("padded", "packed")]
STEPS += [(f"edge dh{128 // c['num_heads']}", p, "packed") for c in EDGE for p in (0.2, 0.5)]
STEPS += [("edge dh32", 0.5, "padded")]


def _users(cfg, B, seed):
    """B histories: the reference's lengths are geometric-ish over 1 .. max_seq_len; a few ids 0 inside them"""
    g = torch.Generator().manual_seed(seed)
    L = cfg["max_seq_len"]
    if L == 200:
        lengths = [(1, 63, 64, 65, 127, 128, 129, 200, 0)[b % 9] for b in range(B)]
    else:
        lengths = torch.randint(1, L + 1, (B,), generator=g).tolist()
        lengths[:3] = [L, 1, L]
    hist = [torch.randint(1, cfg["num_items"] + 1, (n,), generator=g) for n in lengths]
    tgt = [torch.randint(1, cfg["num_items"] + 1, (n,), generator=g) for n in lengths]
    return hist, tgt


def _batches(cfg, B, seed, idle):
    hist, tgt = _users(cfg, B, seed)
    L = max(len(h) for h in hist)
    ids = torch.zeros(B, L, dtype=torch.int64)
    tg = torch.zeros_like(ids)
    for b, (h, t) in enumerate(zip(hist, tgt)):
        if len(h):
            ids[b, L - len(h):], tg[b, L - len(h):] = h, t
    offs = [0]
    for h in hist:
        offs.append(offs[-1] + len(h))
    pids = torch.cat(hist + [torch.zeros(idle, dtype=torch.int64)])
    ptg = torch.cat(tgt + [torch.zeros(idle, dtype=torch.int64)])
    padded = {"input_ids": ids.to(DEV), "targets": tg.to(DEV)}
    packed = {"input_ids": pids.to(DEV), "targets": ptg.to(DEV), "offsets": offs}
    return padded, packed, L


@pytest.mark.parametrize("case", STEPS, ids=_cid)
def test_training_step_vs_fp64(case):
    from genrec_b200.sasrec import SASRec
    from tests.util import frob_relerr, relerr
    shape, p, form = case
    cfg = REFERENCE if shape == "reference" else EDGE[0 if shape == "edge dh32" else 1]
    B = 128 if shape == "reference" else 45
    padded, packed, L = _batches(cfg, B, 5 + int(10 * p), idle=0 if form == "padded" else 41)
    params = sr.seeded_params(cfg, 17)
    m = SASRec(**cfg, dropout=p)
    m.load_state_dict(params, strict=True)
    m = m.to(DEV).train()
    m.return_train_logits = True
    torch.manual_seed(1000 + B + int(10 * p))
    seed = torch.initial_seed() & (2 ** 63 - 1)
    if form == "padded":
        logits, loss = m(padded["input_ids"], padded["targets"])
        batch, shp = padded, ("padded", B, L)
    else:
        T = packed["input_ids"].numel()
        offsets = torch.tensor(packed["offsets"], dtype=torch.int64, device=DEV)
        logits, loss = m.forward_jagged(packed["input_ids"], offsets, cfg["max_seq_len"], packed["targets"])
        batch, shp = packed, ("packed", T, packed["offsets"])
    loss.backward()
    sdv = int(m._seed_dev.item())
    masks = sr.kernel_step_masks(cfg, p, seed, sdv, shp, DEV)
    # the restated layers and seeds are those of the graph's blocks
    cfgs = sorted(_block_cfgs(loss.grad_fn), key=lambda c: c["layer"])
    assert [c["layer"] for c in cfgs] == list(range(cfg["num_blocks"]))
    for c in cfgs:
        assert (c["p"], c["seed"], int(c["seed_dev"].item()), c["apply_mask"]) == (p, seed, sdv, True)
        assert (c["offsets"] is None) == (form == "padded")
    for name, k in sr.mask_sources(masks):                # every source drops something
        assert bool((k == 0).any()), f"mask {name} keeps everything"
    ref = sr.step(params, cfg, batch, masks, form != "padded", device=DEV)
    ac = sr.step(params, cfg, batch, masks, form != "padded", dtype=torch.float32, device=DEV, autocast=True)
    el = abs(loss.item() - ref["loss"].item()) / abs(ref["loss"].item())
    ea = abs(ac["loss"].item() - ref["loss"].item()) / abs(ref["loss"].item())
    rows = [("loss", el, ea, el, ea),
            ("logits", frob_relerr(logits, ref["logits"]), frob_relerr(ac["logits"], ref["logits"]), relerr(logits, ref["logits"]),
             relerr(ac["logits"], ref["logits"]))]
    small = set()
    for name, q in m.named_parameters():
        g, r = q.grad, ref["grads"][name]
        if name.endswith("k_proj.bias"):
            # analytically zero (a shift of a query's scores cancels in the softmax): both sides hold rounding noise alone, which no
            # ratio compares; part A checks the kernel's value, the column sum of its dK, against fp64
            assert bool(torch.isfinite(g).all()), name
            continue
        rows.append((name + ".grad", frob_relerr(g, r), frob_relerr(ac["grads"][name], r), relerr(g, r), relerr(ac["grads"][name], r)))
        if r.numel() < 4096:
            small.add(name + ".grad")
    print(f"\n{_cid(case)}")
    autocast_yardstick(rows, small)


# ------------------------------------------------------------------------------------------------ part C: stand-alone layers
def _sasrec_inputs(B, L, D, seed):
    x = _seeded((B, L, D), seed)
    mask = torch.ones(B, L, 1, device=DEV)
    mask[0, :5] = 0
    return x * mask, mask


def test_multi_head_attention_draws_a_fresh_mask_per_call(monkeypatch):
    from genrec_b200.sasrec import MultiHeadAttention, _AttnFn
    B, L, D, H, p = 4, 65, 64, 2, 0.5
    torch.manual_seed(3)
    attn = MultiHeadAttention(D, H, p).to(DEV).train()
    x, mask = _sasrec_inputs(B, L, D, 1)
    q = x + 0.5
    outs = [attn(q, x, mask) for _ in range(2)]
    assert not torch.equal(outs[0], outs[1]), "two training calls drew the same mask"
    seeds, saved = [], []
    for o in outs:
        Hc, pc, seed, sd = o.grad_fn.cfg
        seeds.append(hr.effective_seed(seed, pc, int(sd.item())))
        saved.append(o.grad_fn.saved_tensors)
        pad, qb, kvb, Q, K, V, att, lse, *_ = saved[-1]
        ref = ar.sasrec_reference(Q, K, V, pad, H, p=p, seed=seeds[-1], layer=0)
        err = ar.errors({"out": att}, ref, ("out",))
        assert not ar.violations(err, "sas"), ar.fmt(err)
        assert torch.equal(o.detach(), att.float() + q)
    assert seeds[0] != seeds[1]
    # backward 1 after forward 2: the core backward re-derives forward 1's mask
    dy = _dy((B, L, D), 9)
    from genrec_b200 import functional as Fn
    spy = Spy(monkeypatch, {Fn: ("sasrec_attention_bwd",)})
    cfg1 = outs[0].grad_fn.cfg
    outs[0].backward(dy)
    (dQ, dK, dV), = spy.take("sasrec_attention_bwd")
    pad, qb, kvb, Q, K, V, att, lse, *_ = saved[0]
    ref = ar.sasrec_reference(Q, K, V, pad, H, dy.bfloat16(), att, p, seeds[0], 0)
    err = ar.errors({"dq": dQ, "dk": dK, "dv": dV}, ref, ("dq", "dk", "dv"))
    assert not ar.violations(err, "sas"), ar.fmt(err)
    # and equals a replay of call 1 with its own seeds, bit for bit
    g1 = {n: t.grad.clone() for n, t in attn.named_parameters()}
    attn.zero_grad(set_to_none=True)
    Hc, pc, seed, sd = cfg1
    o = _AttnFn.apply(q, x, mask, H, p, seed, sd, *[t for _, t in attn.named_parameters()])
    assert torch.equal(o, outs[0])
    o.backward(dy)
    for n, t in attn.named_parameters():
        assert torch.equal(t.grad, g1[n]), n


def test_point_wise_feed_forward_draws_a_fresh_mask_per_call():
    from genrec_b200.sasrec import PointWiseFeedForward, _FfnFn
    T, D, ffn, p = 200, 64, 256, 0.5
    torch.manual_seed(4)
    f = PointWiseFeedForward(D, ffn, p).to(DEV).train()
    x, res = _seeded((T, D), 2), _seeded((T, D), 3)
    outs = [f(x, res) for _ in range(2)]
    assert not torch.equal(outs[0], outs[1]), "two training calls drew the same mask"
    seeds = []
    for y in outs:
        pc, seed, sd = y.grad_fn.cfg
        eff = hr.effective_seed(seed, pc, int(sd.item()))
        seeds.append(eff)
        xb, z1, a1, w1b, w2b = y.grad_fn.saved_tensors
        f1 = dr.linear_forward(xb, w1b, f.fc1.bias.detach(), 2, z1, p, eff, sr.SITE_HID)
        assert torch.equal(a1, f1["a_exact"]), "a1 is not RNE(relu(z1) keep(site 1)) of this call's seeds"
        f2 = dr.linear_residual(a1, w2b, f.fc2.bias.detach(), res, None, p, eff, sr.SITE_OUT)
        assert dr.worst(y.detach(), f2["y"], f2["a_y"]) <= dr.TOL
    assert seeds[0] != seeds[1]
    dy = _dy((T, D), 5)
    pc, seed, sd = outs[0].grad_fn.cfg
    outs[0].backward(dy)
    g1 = {n: t.grad.clone() for n, t in f.named_parameters()}
    f.zero_grad(set_to_none=True)
    y = _FfnFn.apply(x, res, p, seed, sd, f.fc1.weight, f.fc1.bias, f.fc2.weight, f.fc2.bias)
    assert torch.equal(y, outs[0])
    y.backward(dy)
    for n, t in f.named_parameters():
        assert torch.equal(t.grad, g1[n]), n


def test_sasrec_block_draws_a_fresh_mask_per_call(monkeypatch):
    """two calls of a training block without seeds: other masks, each call's stages restated from its own seeds; backward 1 after
    forward 2 re-derives forward 1's masks at every stage"""
    B, L, D, H, p, layer = 5, 65, 64, 2, 0.5, 1
    blk = _block(D, H, p, layer, 21)
    x, mask = _padded_inputs(B, L, D, 22)
    xg = x.clone().requires_grad_(True)
    fs = _fwd_spy(monkeypatch)
    ys = [blk(xg, mask[..., None], _apply_mask=True) for _ in range(2)]
    assert not torch.equal(ys[0], ys[1]), "two training calls drew the same masks"
    calls = fs.take(*["layernorm_fwd"] * 4)
    states, effs = [], []
    for i, y in enumerate(ys):
        qf = calls[2 * i][1]
        cfg = y.grad_fn.cfg
        effs.append(hr.effective_seed(cfg["seed"], cfg["p"], int(cfg["seed_dev"].item())))
        states.append(_forward_items(f"standalone call {i}", y, qf, blk, None, effs[-1]))
    assert effs[0] != effs[1]
    dy = _dy((B, L, D), 23)
    bs = _bwd_spy(monkeypatch)
    ys[0].backward(dy)
    _backward_items("standalone backward 1", blk, states[0], dy, bs, xg.grad, effs[0])


def test_hstu_layer_draws_a_fresh_mask_per_call():
    """two calls of a training HSTULayer without seeds: other masks; each equals the layer run with that call's seeds passed
    explicitly (the path HSTU takes, which tests/test_hstu_block_exact_gpu.py checks against fp64), and backward 1 after forward 2
    gives the gradients of that explicit run, bit for bit"""
    from genrec_b200.hstu import HSTULayer
    B, L, D, H, p = 3, 70, 64, 2, 0.5
    torch.manual_seed(6)
    layer = HSTULayer(D, H, p, 32, 64, 128, True).to(DEV).train()
    g = torch.Generator().manual_seed(7)
    x = torch.randn(B, L, D, generator=g).to(DEV)
    pad = torch.zeros(B, L, dtype=torch.bool)
    pad[0, :9] = True
    ts = (1_300_000_000 + torch.cumsum(torch.randint(1, 10 ** 5, (B, L), generator=g), 1)).to(DEV)
    pad = pad.to(DEV)
    ys = [layer(x, None, pad, ts) for _ in range(2)]
    assert not torch.equal(ys[0], ys[1]), "two training calls drew the same masks"
    cfgs = [y.grad_fn.cfg for y in ys]
    sds = [int(c["seed_dev"].item()) for c in cfgs]
    assert sds[0] != sds[1]
    dy = _dy((B, L, D), 8)
    ys[0].backward(dy)
    g1 = {n: t.grad.clone() for n, t in layer.named_parameters() if t.grad is not None}
    layer.zero_grad(set_to_none=True)
    for i, c in enumerate(cfgs):
        y = layer(x, None, pad, ts, _seed=c["seed"], _seed_dev=torch.tensor([sds[i]], dtype=torch.int64, device=DEV))
        assert torch.equal(y, ys[i]), i
        if i == 0:
            y.backward(dy)
    for n, t in layer.named_parameters():
        if n in g1:
            assert torch.equal(t.grad, g1[n]), n
