"""Packed (jagged) HSTU batches on the H100: pack_jagged against hstu_collate_fn's rows without pads, the packed bias index against
the padded one, one block's packed attention (forward, dQ, dK/dV, bias-table gradients) against the fp64 references of
tests/hstu_block_reference.py, the whole model against the padded batch of the same users, bit-identical repeats, the evaluation
ranks, and a FlatAdam step captured in a CUDA graph and replayed with new offsets, ids and targets."""
import copy

import pytest
import torch

from tests import dense_reference as dr
from tests.hstu_cases import EDGE_LENGTHS, _jagged_model as _model, _users, attention_errors_jagged, run_block_jagged, sign_fix
from tests.util import relerr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
# forward_jagged against forward on the padded batch: the same bf16 operands, the fp32 sums taken over other tile boundaries
MODEL_LOSS_TOL = 2e-3
MODEL_GRAD_TOL = 2e-2


def _collate_rows_without_pads(rows, max_seq_len):
    from genrec_b200.data import hstu_collate_fn
    b = hstu_collate_fn(rows, max_seq_len)
    L = b["input_ids"].shape[1]
    out = {k: [] for k in ("input_ids", "targets", "timestamps")}
    lens = []
    for i, r in enumerate(rows):
        n = min(len(r["history"]), max_seq_len)
        lens.append(n)
        for k in out:
            out[k].append(b[k][i, L - n:])
    return {k: torch.cat(v) for k, v in out.items()}, lens


# ---------------------------------------------------------------------------------------------------- pack_jagged
@pytest.mark.parametrize("max_seq_len", [150, 200])
def test_pack_jagged_is_collate_without_pads(max_seq_len):
    from genrec_b200.data import pack_jagged
    items, ts, off, tgt, rows = _users(EDGE_LENGTHS, 1000, 1)
    ref, lens = _collate_rows_without_pads(rows, max_seq_len)
    total = sum(lens)
    pk = pack_jagged(items, off, tgt, max_seq_len, timestamps=ts)
    assert pk["max_len"] == max(lens) and not bool(pk["overflow"])
    for k in ("input_ids", "targets", "timestamps"):
        assert torch.equal(pk[k].cpu(), ref[k]), k
    exp_off = torch.zeros(len(lens) + 1, dtype=torch.int64)
    exp_off[1:] = torch.cumsum(torch.tensor(lens), 0)
    assert torch.equal(pk["offsets"].cpu(), exp_off)
    # a fixed row count: the packed rows, then idle rows (id 0, target 0, timestamp 0); no host synchronisation needed
    tail = pack_jagged(items, off, tgt, max_seq_len, timestamps=ts, num_tokens=total + 37)
    assert tail["max_len"] == max_seq_len and not bool(tail["overflow"])
    assert torch.equal(tail["offsets"], pk["offsets"])
    for k in ("input_ids", "targets", "timestamps"):
        assert torch.equal(tail[k][:total], pk[k]) and not bool(tail[k][total:].any()), k
    # a batch that does not fit: the flag is raised and the offsets stay inside the rows
    cut = pack_jagged(items, off, tgt, max_seq_len, timestamps=ts, num_tokens=total - 5)
    assert bool(cut["overflow"]) and int(cut["offsets"][-1]) == total - 5
    assert torch.equal(cut["offsets"][:-1], pk["offsets"][:-1])


# ---------------------------------------------------------------------------------------------------- bias index
BIAS_CONFIGS = [("ref", True), ("ref", False), ("fix", True), ("fix", False)]


@pytest.mark.parametrize("pos, timed", BIAS_CONFIGS)
def test_jagged_bias_index_equals_the_padded_rows(pos, timed):
    from genrec_b200.data import collate_jagged, pack_jagged
    from genrec_b200.hstu import HSTULayer
    layer = HSTULayer(64, 2, 0.0, 32, 64, 100, True).to(DEV)
    if pos == "fix":
        sign_fix(layer)
    items, ts, off, tgt, rows = _users(EDGE_LENGTHS, 1000, 2)
    pad_b = collate_jagged(items, off, tgt, 200, timestamps=ts)
    pk = pack_jagged(items, off, tgt, 200, timestamps=ts)
    L = pad_b["input_ids"].shape[1]
    mp = layer._seq_meta((pad_b["input_ids"] == 0).to(torch.uint8), pad_b["timestamps"] if timed else None, L, DEV)
    mj = layer._seq_meta_jagged((pk["input_ids"] == 0).to(torch.uint8), pk["timestamps"] if timed else None, pk["offsets"],
                                pk["max_len"], DEV)
    assert tuple(mj.bias_index.shape) == (int(pk["offsets"][-1]), mj.ld)
    o = pk["offsets"].tolist()
    for b in range(len(rows)):
        n = o[b + 1] - o[b]
        assert torch.equal(mj.bias_index[o[b]:o[b + 1], :n], mp.bias_index[b, L - n:, L - n:L]), b


# ---------------------------------------------------------------------------------------------------- one block, fp64 references


def check_attention_jagged(r):
    worst, excess = attention_errors_jagged(r)
    assert max(worst.values()) <= dr.TOL, worst
    assert all(v <= 1.0 for v in excess.values()), excess


BLOCK_CASES = [
    (EDGE_LENGTHS, 64, 2, ("uni", 0), 64),
    (EDGE_LENGTHS, 128, 4, ("fix", 32, 100), 20),
    (EDGE_LENGTHS, 64, 1, ("fix", 16, 40), "nots"),
    (EDGE_LENGTHS, 128, 2, ("uni", 5), "nots"),
    ([1] * 20 + [2048] + [1] * 10, 128, 4, ("uni", 0), 64),
    ([200], 128, 2, ("fix", 64, 80), 63),
]


@pytest.mark.parametrize("case", BLOCK_CASES, ids=lambda c: f"B{len(c[0])}-max{max(c[0])}-D{c[1]}-dh{c[1] // c[2]}-{c[3][0]}-t{c[4]}")
def test_jagged_attention_vs_fp64(case):
    lengths, D, H, pos, time = case
    check_attention_jagged(run_block_jagged(lengths, D, H, pos, time))


# ---------------------------------------------------------------------------------------------------- the model


def _grads(m):
    return {n: p.grad.detach().clone() for n, p in m.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("fixed", [False, True])
def test_model_matches_the_padded_batch(fixed):
    """forward_jagged's loss and every parameter gradient against forward on collate_jagged of the same users.  The padded batch's last
    pad row predicts the first item from a pad token (hstu_collate_fn's shift); a packed batch has no pad rows, so those targets are
    zeroed on the padded side."""
    from genrec_b200.data import collate_jagged, pack_jagged
    V = 300
    items, ts, off, tgt, _ = _users(EDGE_LENGTHS, V, 3)
    mp = _model(V, fixed=fixed)
    mj = copy.deepcopy(mp)
    pb = collate_jagged(items, off, tgt, 200, timestamps=ts)
    tg = torch.where(pb["input_ids"] == 0, 0, pb["targets"])
    _, lp = mp(pb["input_ids"], pb["timestamps"], tg)
    lp.backward()
    pk = pack_jagged(items, off, tgt, 200, timestamps=ts, num_tokens=sum(EDGE_LENGTHS) + 23)
    _, lj = mj.forward_jagged(pk["input_ids"], pk["offsets"], pk["max_len"], pk["timestamps"], pk["targets"])
    lj.backward()
    assert abs(lj.item() - lp.item()) <= MODEL_LOSS_TOL * abs(lp.item()), (lj.item(), lp.item())
    gp, gj = _grads(mp), _grads(mj)
    assert gp.keys() == gj.keys()
    errs = {n: relerr(gj[n], gp[n]) for n in gp}
    assert max(errs.values()) <= MODEL_GRAD_TOL, errs


def _jagged_step(m, pk, ids=None):
    for p in m.parameters():
        p.grad = None
    _, loss = m.forward_jagged(pk["input_ids"] if ids is None else ids, pk["offsets"], pk["max_len"], pk["timestamps"], pk["targets"])
    loss.backward()
    return loss.detach().clone(), _grads(m)


def test_idle_rows_and_repeats_change_no_bit():
    """Two identical packed steps give the same bits; so does a step whose idle rows (past offsets[B]) hold other ids."""
    from genrec_b200.data import pack_jagged
    V = 300
    items, ts, off, tgt, _ = _users(EDGE_LENGTHS, V, 4)
    total = sum(EDGE_LENGTHS)
    pk = pack_jagged(items, off, tgt, 200, timestamps=ts, num_tokens=total + 40)
    m = _model(V)
    ids = pk["input_ids"].clone()
    ids[total:] = torch.arange(1, 41, device=DEV)
    l1, g1 = _jagged_step(m, pk, ids)
    l2, g2 = _jagged_step(m, pk, ids)
    assert torch.equal(l1, l2) and all(torch.equal(g1[n], g2[n]) for n in g1)
    ids[total:] = torch.arange(1, 41, device=DEV).flip(0)       # the idle rows' ids, permuted: the embedding's sort runs stay put
    l3, g3 = _jagged_step(m, pk, ids)
    assert torch.equal(l1, l3) and all(torch.equal(g1[n], g3[n]) for n in g1)
    l4, g4 = _jagged_step(m, pk)                                # idle ids 0: only the item table's summation runs may move
    assert torch.equal(l1, l4)
    assert all(torch.equal(g1[n], g4[n]) for n in g1 if n != "item_embedding.weight")
    assert relerr(g4["item_embedding.weight"], g1["item_embedding.weight"]) <= 1e-5


@pytest.mark.parametrize("with_exclude", [False, True])
def test_evaluate_batch_jagged_ranks(with_exclude):
    import genrec_b200.functional as Fn
    from genrec_b200.data import pack_jagged
    V = 300
    items, ts, off, tgt, _ = _users(EDGE_LENGTHS, V, 5)
    m = _model(V).eval()
    pk = pack_jagged(items, off, tgt, 200, timestamps=ts)
    B = len(EDGE_LENGTHS)
    exclude = torch.randint(1, V + 1, (B, 12), device=DEV) if with_exclude else None
    metrics, ranks = m.evaluate_batch_jagged(pk["input_ids"], pk["offsets"], pk["max_len"], pk["timestamps"], tgt, exclude=exclude,
                                             want_ranks=True)
    with torch.no_grad():
        x = m.encode_jagged(pk["input_ids"], pk["offsets"], pk["max_len"], pk["timestamps"])
    o = pk["offsets"]
    last = x[(o[1:] - 1).clamp(min=0)]
    logits = Fn.head_logits(last[:, None], m.final_norm.weight, m.final_norm.bias, m.item_embedding.weight, m._table_mirror(),
                            m.final_norm.eps)[:, 0]
    if exclude is not None:
        logits = logits.scatter(1, exclude, float("-inf"))
    ref_tg = torch.where(o[1:] > o[:-1], tgt, 0)
    if exclude is not None:
        ref_tg = torch.where((exclude == tgt[:, None]).any(1), 0, ref_tg)
    _, ref_ranks = Fn.eval_rank_metrics(logits, ref_tg, want_ranks=True)
    ref_ranks = torch.where(ref_tg > 0, ref_ranks, 0)
    assert torch.equal(ranks, ref_ranks), (ranks, ref_ranks)
    assert int(ranks[0]) == 0                                  # the empty history is not ranked


def test_captured_step_follows_rewritten_offsets_ids_and_targets():
    """FlatAdam(unit_loss_grad=True, lazy_table=True): a packed training step captured in a CUDA graph, replayed with new offsets,
    ids, timestamps and targets at fixed (B, T, max_len), gives the eager steps' bits."""
    from genrec_b200.data import pack_jagged
    from genrec_b200.optim import FlatAdam
    V, B, T, max_len = 300, 9, 1850, 200
    draws = []
    for k in range(6):
        g = torch.Generator().manual_seed(100 + k)
        lengths = torch.randint(0, 201, (B,), generator=g).tolist()
        items, ts, off, tgt, _ = _users(lengths, V, 200 + k)
        pk = pack_jagged(items, off, tgt, max_len, timestamps=ts, num_tokens=T)
        assert not bool(pk["overflow"])
        draws.append(tuple(pk[n] for n in ("input_ids", "offsets", "timestamps", "targets")))

    def run(captured):
        m = _model(V, blocks=2)
        opt = FlatAdam(m, lr=1e-3, unit_loss_grad=True, lazy_table=True)
        bufs = [t.clone() for t in draws[0]]

        def load(i):
            for dst, src in zip(bufs, draws[i]):
                dst.copy_(src)

        def step():
            ids, off, ts, tg = bufs
            _, loss = m.forward_jagged(ids, off, max_len, ts, tg)
            loss.backward()
            opt.step()
            return loss

        losses = []
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for i in range(3):
                load(i)
                losses.append(step().item())
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        if captured:
            graph = torch.cuda.CUDAGraph()
            load(3)
            with torch.cuda.graph(graph):
                loss = step()
            for i in range(3, 6):
                load(i)
                graph.replay()
                losses.append(loss.item())
        else:
            for i in range(3, 6):
                load(i)
                losses.append(step().item())
        return losses, torch.cat([opt.flat, opt.m, opt.v])

    eager, s_eager = run(False)
    graphed, s_graph = run(True)
    assert eager == graphed, (eager, graphed)
    assert torch.equal(s_eager, s_graph)
