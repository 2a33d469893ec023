"""Packed (jagged) SASRec batches on the H100: the packed attention (forward, dQ, dK/dV) against the fp64 reference of
tests/attention_reference.py per sequence under dropout, device offsets out of contract, the packed embedding and its position rule
against tests/dense_reference.py, the packed position gradient bit for bit against the padded one, the whole model against the
padded batch of the same users and against the oracle, the evaluation ranks, bit-identical repeats, a training step captured in a
CUDA graph and replayed with new offsets, ids and targets, and the sampled head.

Packed dropout rule (restated from csrc/attn_sasrec.cuh): the attention mask of query i of a sequence whose first token row is tok0,
head h, key j (its index within the sequence) has row key (tok0 + i) * H + h and column j, at site 8 layer + 3.  The embedding's mask
is keyed by the token row and the column, at site 250."""
import copy
import ctypes as C
import math

import numpy as np
import pytest
import torch

from tests import attention_reference as ar
from tests import dense_reference as dr
from tests.util import relerr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
EDGE_LENGTHS = [0, 1, 63, 64, 65, 127, 128, 129, 200]
MAX_LEN = 200
# forward_jagged against forward on the padded batch: the same bf16 operands, the fp32 sums taken over other tile boundaries
MODEL_LOSS_TOL = 2e-3
MODEL_GRAD_TOL = 2e-2


# ---------------------------------------------------------------------------------------------------- attention
def packed_keep(tok0, n, H, p, seed, site, device="cpu"):
    """[1, H, n, n] keep-scale matrix of the packed rule: row key (tok0 + i) H + h, column j."""
    rows = (tok0 + np.arange(n, dtype=np.int64))[None, :] * H + np.arange(H, dtype=np.int64)[:, None]   # [H, n]
    drop = ar.drop_mask(rows.reshape(-1) & 0xFFFFFFFF, n, p, seed, site)
    return torch.from_numpy(np.where(drop, 0.0, ar.keep_scale(p)[1])).view(1, H, n, n).to(device)


def packed_reference(Q, K, V, pad, H, dO, O, p, seed, layer, tok0):
    """sasrec_reference on one sequence [1, n, D] with the packed dropout rule in place of the padded one."""
    orig = ar.attn_keep
    ar.attn_keep = lambda B, H_, Lq, Lk, p_, seed_, site, device="cpu": packed_keep(tok0, Lq, H_, p_, seed_, site, device)
    try:
        return ar.sasrec_reference(Q, K, V, pad, H, dO, O, p, seed, layer)
    finally:
        ar.attn_keep = orig


def _batch(lengths, D, lead, tail, seed):
    g = torch.Generator().manual_seed(seed)
    T = lead + sum(lengths) + tail
    off = torch.tensor([lead] + [lead + int(s) for s in np.cumsum(lengths)], dtype=torch.int64)
    Q, K, V, dO = [(0.7 * torch.randn(T, D, generator=g)).bfloat16().to(DEV) for _ in range(4)]
    pad = (torch.rand(T, generator=g) < 0.04).to(torch.uint8)           # id-0 tokens inside the sequences
    pad[:lead] = 1
    pad[T - tail:] = 1
    return T, off.to(DEV), Q, K, V, dO, pad.to(DEV)


def _check_attention(lengths, dh, H, p, use_seed_dev, lead, tail, seed=11, layer=1):
    D = H * dh
    T, off, Q, K, V, dO, pad = _batch(lengths, D, lead, tail, seed)
    s0, s1 = 0x1234_5678_9ABC, 977
    sd = torch.tensor([s1], dtype=torch.int64, device=DEV) if use_seed_dev else None
    eff = (s0 + s1) if use_seed_dev else s0
    import genrec_b200.functional as Fn
    out, lse = Fn.sasrec_attention_fwd(Q, K, V, pad, H, p, s0, sd, layer, off, MAX_LEN)
    dq, dk, dv = Fn.sasrec_attention_bwd(Q, K, V, pad, out, lse, dO, H, p, s0, sd, layer, off, MAX_LEN)
    torch.cuda.synchronize()
    worst = {}
    o = off.tolist()
    for b, n in enumerate(lengths):
        if n == 0:
            continue
        s = slice(o[b], o[b] + n)
        ref = packed_reference(Q[s][None], K[s][None], V[s][None], pad[s][None], H, dO[s][None], out[s][None], p, eff, layer, o[b])
        got = {"out": out[s][None], "dq": dq[s][None], "dk": dk[s][None], "dv": dv[s][None], "lse": lse[:, s][None]}
        err = ar.errors(got, ref, ("out", "dq", "dk", "dv"))
        bad = ar.violations(err, "sas") + ar.sasrec_exact(got, ref)
        assert not bad, (n, bad, ar.fmt(err))
        for k, (w, _) in err.items():
            worst[k] = max(worst.get(k, 0.0), w)
    idle = torch.ones(T, dtype=torch.bool, device=DEV)
    idle[o[0]:o[-1]] = False
    for name, t in (("O", out), ("dQ", dq), ("dK", dk), ("dV", dv)):
        assert bool((t[idle] == 0).all()), f"an idle row of {name} is not exactly 0"
    print(f"\nsasrec packed dh={dh} p={p} seed_dev={use_seed_dev} lead={lead} tail={tail} T={T} worst {worst}")


# layouts: extra sequence lengths, leading idle rows, trailing idle rows.  sum(EDGE_LENGTHS) = 777 = 9 (mod 128)
LAYOUTS = {"T=1 mod 128": ([120], 0, 0), "T=127 mod 128": ([118], 0, 0), "idle, T=1 mod 128": ([], 0, 120),
           "idle, T=127 mod 128": ([], 0, 118), "leading idle rows": ([], 3, 5)}


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("p", [0.0, 0.2, 0.5])
@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("use_seed_dev", [False, True])
def test_packed_attention_vs_fp64(layout, p, dh, use_seed_dev):
    extra, lead, tail = LAYOUTS[layout]
    if p == 0.0 and use_seed_dev:
        pytest.skip("seed_dev only moves the dropout masks")
    _check_attention(EDGE_LENGTHS + extra, dh, 2, p, use_seed_dev, lead, tail)


@pytest.mark.parametrize("p", [0.0, 0.5])
def test_packed_attention_only_idle_rows(p):
    """Every sequence empty: O and dQ | dK | dV are exactly zero on all T rows."""
    _check_attention([0, 0, 0, 0], 64, 2, p, False, 0, 64)


def _sas_dims(B, D, H, p=0.0, seed=0, layer=0):
    from genrec_b200._lib import SasrecDims
    return SasrecDims(B, MAX_LEN, D, H, float(p), seed, None, layer)


def test_device_offsets_past_T_write_nothing_past_T():
    """offsets[B] = T + 40: the kernels clamp the last sequence to T, write nothing into 64 canary rows past T (nor past lse's H T
    entries), and every row below T has the bits of the well-formed batch."""
    from genrec_b200._lib import check, load, ptr
    lib = load()
    H, D, p = 2, 128, 0.2
    lengths = EDGE_LENGTHS
    T, off, Q, K, V, dO, pad = _batch(lengths, D, 0, 64, 21)     # 64 rows past the sequences: the canaries
    T -= 64
    bad = off.clone()
    bad[-1] = T + 40
    dims = _sas_dims(len(lengths), D, H, p, 77)

    def run(o):
        out = torch.full((T + 64, D), 3.0, dtype=torch.bfloat16, device=DEV)
        lse = torch.full((H * T + 64,), 3.0, device=DEV)
        grads = [torch.full((T + 64, D), 3.0, dtype=torch.bfloat16, device=DEV) for _ in range(3)]
        check(lib.grb_sasrec_attention_forward_jagged(C.byref(dims), ptr(o), T, ptr(Q), ptr(K), ptr(V), ptr(pad), ptr(out), ptr(lse), None))
        check(lib.grb_sasrec_attention_backward_jagged(C.byref(dims), ptr(o), T, ptr(Q), ptr(K), ptr(V), ptr(pad), ptr(out), ptr(lse),
                                                       ptr(dO), *[ptr(g) for g in grads], None))
        torch.cuda.synchronize()
        return out, lse, grads

    out_b, lse_b, g_b = run(bad)
    out_g, lse_g, g_g = run(off)
    for t in (out_b, *g_b):
        assert bool((t[T:] == 3.0).all()), "a row past T was written"
    assert bool((lse_b[H * T:] == 3.0).all())
    assert torch.equal(out_b[:T], out_g[:T]) and torch.equal(lse_b[:H * T], lse_g[:H * T])
    assert all(torch.equal(a[:T], b[:T]) for a, b in zip(g_b, g_g))


# ---------------------------------------------------------------------------------------------------- embedding
def _positions(off, max_len):
    """The position rule on the host: (position of each row or -1, P)."""
    o = off.tolist()
    lens = [min(b - a, max_len) for a, b in zip(o, o[1:])]
    P = max(lens)
    pos = [-1] * o[0]
    for n in lens:
        pos += [P - n + i for i in range(n)]
    return pos, P


@pytest.mark.parametrize("p", [0.0, 0.2])
def test_packed_embedding_vs_fp64(p):
    """x = drop(E[id] sqrt(D) + pos[P - n + i]) * (id != 0) on the sequence rows, exact zeros on the idle rows; dE and dpos of a
    random dx against fp64, with the masks keyed by token row."""
    import genrec_b200.functional as Fn
    g = torch.Generator().manual_seed(5)
    V, D, max_len, idle = 300, 64, 50, 13
    lengths = [0, 1, 5, 50, 17, 3, 31]
    T = sum(lengths) + idle
    off = torch.tensor([0] + np.cumsum(lengths).tolist(), dtype=torch.int64)
    ids = torch.randint(1, V + 1, (T,), generator=g)
    ids[[2, 9, 40]] = 0                                   # id 0 inside sequences
    ids[T - idle:] = torch.randint(1, V + 1, (idle,), generator=g)   # idle rows holding real ids still give x = 0
    E = torch.randn(V + 1, D, generator=g)
    E[0] = 0
    pos = torch.randn(max_len, D, generator=g)
    seed, scale = 4321, math.sqrt(D)
    Eg, posg = E.to(DEV).requires_grad_(True), pos.to(DEV).requires_grad_(True)
    x, pad = Fn.EmbedFn.apply(ids.to(DEV), Eg, posg, scale, 1, p, seed, None, None, off.to(DEV), max_len)
    dx = torch.randn(T, D, generator=g)
    x.backward(dx.to(DEV))
    positions, P = _positions(off, max_len)
    positions += [-1] * idle
    prow = torch.tensor(positions)
    live_rows = prow >= 0
    assert torch.equal(pad.cpu().bool(), ~live_rows | (ids == 0))
    assert bool((x[~live_rows.to(DEV)] == 0).all())
    fwd = dr.embed_forward(ids.view(1, T), E, pos[prow.clamp(min=0)], T, scale, 1, p, seed)   # row t takes position row prow[t]
    err = {"x": dr.worst(x[live_rows.to(DEV)], fwd["x"][live_rows], fwd["a_x"][live_rows])}
    # dE: the token rows with their own masks; the idle rows take no gradient
    ids_live = torch.where(live_rows, ids, 0)
    bwd = dr.embed_backward(ids_live.view(1, T), dx, T, V + 1, 0, scale, 1, p, seed)
    err["dE"] = dr.worst(Eg.grad, bwd["dE"], bwd["a_dE"])
    km = dr.keep(range(T), D, p, seed, dr.SITE_EMBED)
    t = dx.double() * km
    t[~live_rows | (ids == 0)] = 0
    dpos = torch.zeros(max_len, D, dtype=torch.float64).index_add_(0, prow.clamp(min=0), t)
    magp = torch.zeros(max_len, D, dtype=torch.float64).index_add_(0, prow.clamp(min=0), t.abs())
    err["dpos"] = dr.worst(posg.grad, dpos, (len(lengths) + 2) * dr.C * magp + dr.C * dpos.abs())
    assert bool((posg.grad[P:] == 0).all())
    assert not dr.violations(err), dr.fmt(err)


def test_packed_dpos_is_bit_identical_to_the_padded_batch():
    """dx of a left-padded batch gathered to the packed rows: the packed position gradient sums the same terms in the same order as
    grb_embed_backward on the padded batch, so the two are equal bit for bit."""
    import genrec_b200.functional as Fn
    g = torch.Generator().manual_seed(6)
    V, D, max_len = 300, 64, 50
    lengths = [0, 1, 5, 50, 17, 3, 50, 49] * 40
    B, P = len(lengths), max(lengths)
    T = sum(lengths)
    ids_pad = torch.zeros(B, P, dtype=torch.int64)
    for b, n in enumerate(lengths):
        ids_pad[b, P - n:] = torch.randint(1, V + 1, (n,), generator=g)
    ids_pad[3, P - 2] = 0                                 # an id 0 inside a sequence
    real = torch.zeros(B, P, dtype=torch.bool)
    for b, n in enumerate(lengths):
        real[b, P - n:] = True
    ids = ids_pad[real]
    off = torch.tensor([0] + np.cumsum(lengths).tolist(), dtype=torch.int64, device=DEV)
    E = torch.randn(V + 1, D, generator=g, device="cpu").to(DEV)
    dx_pad = torch.randn(B, P, D, generator=g).to(DEV)
    pos_a = torch.randn(max_len, D, generator=g).to(DEV).requires_grad_(True)
    pos_b = pos_a.detach().clone().requires_grad_(True)
    x, _ = Fn.EmbedFn.apply(ids_pad.to(DEV), E, pos_a, math.sqrt(D), 1, 0.0, 0, None)
    x.backward(dx_pad)
    xj, _ = Fn.EmbedFn.apply(ids.to(DEV), E, pos_b, math.sqrt(D), 1, 0.0, 0, None, None, off, max_len)
    xj.backward(dx_pad[real.to(DEV)])
    assert torch.equal(xj, x[real.to(DEV)])
    assert torch.equal(pos_a.grad, pos_b.grad)


@pytest.mark.parametrize("num_tokens", [None, 400])
def test_positions_follow_rewritten_device_offsets(num_tokens):
    """P is derived on the device: rewriting the offsets in place (same T, same host max_len) moves every token's position."""
    import genrec_b200.functional as Fn
    from genrec_b200.data import pack_jagged
    g = torch.Generator().manual_seed(7)
    V, D, msl = 300, 64, 50
    E = torch.randn(V + 1, D, generator=g).to(DEV)
    pos = torch.randn(msl, D, generator=g).to(DEV)
    batches = [[3, 12, 7], [30, 2, 9], [50, 50, 1], [1, 1, 61]]
    first = None
    for lengths in batches:
        items = torch.randint(1, V + 1, (sum(lengths),), generator=g).to(DEV)
        off = torch.tensor([0] + np.cumsum(lengths).tolist(), dtype=torch.int64, device=DEV)
        pk = pack_jagged(items, off, torch.ones(3, dtype=torch.int64, device=DEV), msl, num_tokens=num_tokens or sum(min(n, msl) for n in lengths))
        if first is None:
            first = pk
            T, max_len = pk["input_ids"].numel(), (pk["max_len"] if num_tokens else msl)
        else:
            n = min(pk["input_ids"].numel(), T)
            first["input_ids"].zero_()
            first["input_ids"][:n].copy_(pk["input_ids"][:n])
            first["offsets"].copy_(pk["offsets"].clamp(max=T))
        x, _ = Fn.EmbedFn.apply(first["input_ids"], E, pos, math.sqrt(D), 1, 0.0, 0, None, None, first["offsets"], max_len)
        prow, P = _positions(first["offsets"].cpu(), max_len)
        prow = torch.tensor(prow + [-1] * (T - len(prow)), device=DEV)
        ids = first["input_ids"]
        want = torch.where((prow >= 0)[:, None], E[ids] * np.float32(math.sqrt(D)) + pos[prow.clamp(min=0)], 0.0) * (ids != 0)[:, None]
        torch.testing.assert_close(x, want, rtol=1e-6, atol=1e-6)


# ---------------------------------------------------------------------------------------------------- the model
MODEL_LENGTHS = [0, 1, 3, 9, 50, 61, 17, 2, 33, 50]


def _model(V, blocks=2):
    from genrec_b200.sasrec import SASRec
    torch.manual_seed(0)
    return SASRec(V, 50, 64, 2, blocks, 256, dropout=0.0).to(DEV).train()


def _users(lengths, V, seed):
    g = torch.Generator().manual_seed(seed)
    hist = [torch.randint(1, V + 1, (n,), generator=g) for n in lengths]
    tgt = torch.randint(1, V + 1, (len(lengths),), generator=g)
    offsets = torch.zeros(len(lengths) + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(torch.tensor(lengths, dtype=torch.int64), 0)
    return torch.cat(hist).long().to(DEV), offsets.to(DEV), tgt.to(DEV)


def _grads(m):
    return {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}


def test_model_matches_the_padded_batch():
    """forward_jagged's loss and every parameter gradient (position_embedding.weight included) against forward on collate_jagged
    of the same users, the pad rows' targets zeroed on the padded side (the shift gives the last pad row a target)."""
    from genrec_b200.data import collate_jagged, pack_jagged
    V = 300
    items, off, tgt = _users(MODEL_LENGTHS, V, 3)
    mp = _model(V)
    mj = copy.deepcopy(mp)
    pb = collate_jagged(items, off, tgt, 50)
    tg = torch.where(pb["input_ids"] == 0, 0, pb["targets"])
    _, lp = mp(pb["input_ids"], tg)
    lp.backward()
    pk = pack_jagged(items, off, tgt, 50, num_tokens=sum(min(n, 50) for n in MODEL_LENGTHS) + 23)
    _, lj = mj.forward_jagged(pk["input_ids"], pk["offsets"], 50, pk["targets"])
    lj.backward()
    assert abs(lj.item() - lp.item()) <= MODEL_LOSS_TOL * abs(lp.item()), (lj.item(), lp.item())
    gp, gj = _grads(mp), _grads(mj)
    assert gp.keys() == gj.keys() and "position_embedding.weight" in gj
    errs = {n: relerr(gj[n], gp[n]) for n in gp if gp[n].abs().max() > 0}
    assert max(errs.values()) <= MODEL_GRAD_TOL, errs


def test_forward_jagged_vs_oracle():
    """forward_jagged's loss and logits against the CPU oracle on the left-padded batch, at test_cfg1_shape_vs_oracle's tolerance."""
    from genrec_b200.data import collate_jagged, pack_jagged
    from oracle import sasrec as osr
    V = 1000
    items, off, tgt = _users(MODEL_LENGTHS, V, 8)
    m = _model(V)
    sd = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    pb = collate_jagged(items, off, tgt, 50)
    tg = torch.where(pb["input_ids"] == 0, 0, pb["targets"])
    lo, ls = osr.sasrec_forward(pb["input_ids"].cpu(), tg.cpu(), sd, 2, 2)
    m.return_train_logits = True
    pk = pack_jagged(items, off, tgt, 50)
    lg, lsg = m.forward_jagged(pk["input_ids"], pk["offsets"], pk["max_len"], pk["targets"])
    assert abs(lsg.item() - ls.item()) < 2e-2
    real = (pb["input_ids"] != 0).cpu()
    assert relerr(lg.detach().cpu(), lo.detach()[real]) < 4e-2


def _jagged_step(m, pk, ids=None):
    for p in m.parameters():
        p.grad = None
    _, loss = m.forward_jagged(pk["input_ids"] if ids is None else ids, pk["offsets"], pk["max_len"], pk["targets"])
    loss.backward()
    return loss.detach().clone(), _grads(m)


def test_idle_rows_and_repeats_change_no_bit():
    """Two identical packed steps give the same bits, and so does a step whose idle rows (past offsets[B]) hold other ids."""
    from genrec_b200.data import pack_jagged
    V = 300
    items, off, tgt = _users(MODEL_LENGTHS, V, 4)
    total = sum(min(n, 50) for n in MODEL_LENGTHS)
    pk = pack_jagged(items, off, tgt, 50, num_tokens=total + 40)
    m = _model(V)
    l1, g1 = _jagged_step(m, pk)
    l2, g2 = _jagged_step(m, pk)
    assert torch.equal(l1, l2) and all(torch.equal(g1[n], g2[n]) for n in g1)
    ids = pk["input_ids"].clone()
    ids[total:] = torch.arange(1, 41, device=DEV)
    l3, g3 = _jagged_step(m, pk, ids)
    assert torch.equal(l1, l3) and all(torch.equal(g1[n], g3[n]) for n in g1)


@pytest.mark.parametrize("with_exclude", [False, True])
def test_evaluate_batch_jagged_ranks(with_exclude):
    import genrec_b200.functional as Fn
    from genrec_b200.data import pack_jagged
    V = 300
    items, off, tgt = _users(MODEL_LENGTHS, V, 5)
    m = _model(V).eval()
    pk = pack_jagged(items, off, tgt, 50)
    B = len(MODEL_LENGTHS)
    exclude = torch.randint(1, V + 1, (B, 12), device=DEV) if with_exclude else None
    metrics, ranks = m.evaluate_batch_jagged(pk["input_ids"], pk["offsets"], pk["max_len"], tgt, exclude=exclude, want_ranks=True)
    with torch.no_grad():
        x = m.encode_jagged(pk["input_ids"], pk["offsets"], pk["max_len"])
    o = pk["offsets"]
    last = x[(o[1:] - 1).clamp(min=0)]
    logits = Fn.head_logits(last[:, None], m.final_norm.weight, m.final_norm.bias, m.item_embedding.weight,
                            Fn.cast_bf16(m.item_embedding.weight), m.final_norm.eps)[:, 0]
    if exclude is not None:
        logits = logits.scatter(1, exclude, float("-inf"))
    ref_tg = torch.where(o[1:] > o[:-1], tgt, 0)
    if exclude is not None:
        ref_tg = torch.where((exclude == tgt[:, None]).any(1), 0, ref_tg)
    ref_metrics, ref_ranks = Fn.eval_rank_metrics(logits, ref_tg, want_ranks=True)
    ref_ranks = torch.where(ref_tg > 0, ref_ranks, 0)
    assert torch.equal(ranks, ref_ranks), (ranks, ref_ranks)
    assert int(ranks[0]) == 0                                  # the empty history is not ranked
    torch.testing.assert_close(metrics, ref_metrics)


def test_captured_step_follows_rewritten_offsets_ids_and_targets():
    """torch Adam(capturable=True): a packed training step captured in a CUDA graph at fixed (B, T, max_len), replayed with new
    offsets, ids and targets whose longest history (P) changes between replays, gives the eager steps' bits."""
    from genrec_b200.data import pack_jagged
    V, B, T, max_len = 300, 16, 600, 50
    draws, longest = [], []
    for k in range(6):
        g = torch.Generator().manual_seed(100 + k)
        lengths = torch.randint(0, 10 + 8 * k, (B,), generator=g).clamp(max=50).tolist()
        items, off, tgt = _users(lengths, V, 200 + k)
        pk = pack_jagged(items, off, tgt, max_len, num_tokens=T)
        assert not bool(pk["overflow"])
        draws.append(tuple(pk[n] for n in ("input_ids", "offsets", "targets")))
        longest.append(max(lengths))
    assert len(set(longest[3:])) == 3

    def run(captured):
        m = _model(V)
        opt = torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True)
        bufs = [t.clone() for t in draws[0]]

        def load(i):
            for dst, src in zip(bufs, draws[i]):
                dst.copy_(src)

        def step():
            ids, off, tg = bufs
            _, loss = m.forward_jagged(ids, off, max_len, tg)
            loss.backward()
            opt.step()
            return loss

        losses = []
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for i in range(3):
                load(i)
                opt.zero_grad(set_to_none=True)
                losses.append(step().item())
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        if captured:
            graph = torch.cuda.CUDAGraph()
            load(3)
            opt.zero_grad(set_to_none=True)
            with torch.cuda.graph(graph):
                loss = step()
            for i in range(3, 6):
                load(i)
                graph.replay()
                losses.append(loss.item())
        else:
            for i in range(3, 6):
                load(i)
                opt.zero_grad(set_to_none=True)
                losses.append(step().item())
        return losses, torch.cat([p.detach().reshape(-1) for p in m.parameters()])

    eager, s_eager = run(False)
    graphed, s_graph = run(True)
    assert eager == graphed, (eager, graphed)
    assert torch.equal(s_eager, s_graph)


def test_sampled_head_through_forward_jagged():
    """forward_jagged with negatives is the sampled head on encode_jagged's rows (bit for bit), and matches the padded model's sampled
    loss to rounding."""
    import genrec_b200.functional as Fn
    from genrec_b200.data import collate_jagged, pack_jagged, sample_negatives
    V = 300
    items, off, tgt = _users(MODEL_LENGTHS, V, 9)
    m = _model(V)
    probs = (torch.rand(V + 1, generator=torch.Generator().manual_seed(1)) + 0.1).to(DEV)
    neg, log_q = sample_negatives(V, 64, probs=probs, generator=torch.Generator(device=DEV).manual_seed(1))
    pk = pack_jagged(items, off, tgt, 50)
    T = pk["input_ids"].numel()
    _, loss = m.forward_jagged(pk["input_ids"], pk["offsets"], pk["max_len"], pk["targets"], negatives=neg, log_q=log_q)
    with torch.no_grad():
        x = m.encode_jagged(pk["input_ids"], pk["offsets"], pk["max_len"])
        ref = Fn.SampledHeadLossFn.apply(x.view(1, T, -1), m.final_norm.weight, m.final_norm.bias, m.item_embedding.weight,
                                         Fn.cast_bf16(m.item_embedding.weight), pk["targets"].view(1, T), neg, log_q, m.final_norm.eps)
    assert torch.equal(loss.detach(), ref)
    pb = collate_jagged(items, off, tgt, 50)
    _, lp = m(pb["input_ids"], torch.where(pb["input_ids"] == 0, 0, pb["targets"]), negatives=neg, log_q=log_q)
    assert abs(loss.item() - lp.item()) <= MODEL_LOSS_TOL * abs(lp.item())
