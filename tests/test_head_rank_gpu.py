"""grb_head_rank (Fn.head_rank_metrics, HSTU.evaluate_batch, SASRec.evaluate_batch) against the logits path: head_logits of the same
rows followed by eval_rank_metrics.  Ranks and hit counts must match exactly, because the fused sweep accumulates every score,
the target's included, as the logits GEMM does; the NDCG sums may differ by the order of the float atomics."""
import math

import pytest
import torch

import genrec_b200.functional as Fn

pytestmark = pytest.mark.gpu

EPS = 1e-5
NEG = float("-inf")


def _head(R, D, C, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R, D, generator=g).cuda()
    ln_g = (1 + 0.1 * torch.randn(D, generator=g)).cuda()
    ln_b = (0.1 * torch.randn(D, generator=g)).cuda()
    tb = (0.05 * torch.randn(C, D, generator=g)).to(torch.bfloat16).cuda()
    return x, ln_g, ln_b, tb


def _logits(x, ln_g, ln_b, tb):
    return Fn.head_logits(x[:, None, :], ln_g, ln_b, tb, tb, EPS)[:, 0, :]


def _targets(R, C, seed):
    """random ids in 1..C-1, with 0, 1, C-1, C, C+7 and negative ids at the start and the end of the batch"""
    g = torch.Generator().manual_seed(seed)
    tg = torch.randint(1, C, (R,), generator=g)
    special = torch.tensor([0, 1, C - 1, C, C + 7, -3, -(1 << 40)])
    n = min(R, len(special))
    tg[:n] = special[:n]
    if R > 2 * len(special):
        tg[-n:] = special[torch.randperm(len(special), generator=g)][:n]
    return tg.cuda()


def _assert_same(got, ref):
    (m, r), (rm, rr) = got, ref
    assert torch.equal(r, rr), ((r != rr).nonzero()[:8], r[r != rr][:8], rr[r != rr][:8])
    assert torch.equal(m[:3], rm[:3]), (m, rm)
    torch.testing.assert_close(m[3:], rm[3:], rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------ 1. the logits path, exactly
@pytest.mark.parametrize("C", [2, 3, 127, 128, 129, 12102, 1000001])
@pytest.mark.parametrize("D", [64, 128, 256])
def test_ranks_equal_the_logits_path(D, C):
    for R in (1, 127, 128, 129, 1000):
        x, ln_g, ln_b, tb = _head(R, D, C, seed=R + D + C)
        tg = _targets(R, C, seed=R * 7 + C)
        got = Fn.head_rank_metrics(x, ln_g, ln_b, tb, EPS, tg, want_ranks=True)
        ref = Fn.eval_rank_metrics(_logits(x, ln_g, ln_b, tb), tg, want_ranks=True)
        _assert_same(got, ref)
        ok = (tg >= 1) & (tg < C)
        assert torch.equal(got[1] == 0, ~ok)
        del x, tb


# ------------------------------------------------------------------------------------------------ 2. exact ties
@pytest.mark.parametrize("D", [64, 128, 256])
def test_exact_ties_count_only_lower_ids(D):
    R, C = 300, 3001
    x, ln_g, ln_b, tb = _head(R, D, C, seed=D)
    lg = _logits(x, ln_g, ln_b, tb)
    top = lg[:, 1:].argmax(1) + 1                       # each row's best item (lowest id among equal maxima)
    got = Fn.head_rank_metrics(x, ln_g, ln_b, tb, EPS, top, want_ranks=True)[1]
    assert (got == 1).all()                             # a target that scores the maximum has rank 1
    # rows whose best items are distinct and at least 3 apart: copy the target's table row to ids t - 1 and t + 1
    rows, taken = [], set()
    for r, t in enumerate(top.tolist()):
        if 2 <= t <= C - 2 and not any(abs(t - u) <= 2 for u in taken):
            rows.append(r)
            taken.add(t)
        if len(rows) == 24:
            break
    assert len(rows) >= 12
    tb2 = tb.clone()
    for r in rows:
        t = int(top[r])
        tb2[t - 1] = tb[t]
        tb2[t + 1] = tb[t]
    tg = torch.randint(1, C, (R,), device="cuda")
    tg[rows] = top[rows]
    m, ranks = Fn.head_rank_metrics(x, ln_g, ln_b, tb2, EPS, tg, want_ranks=True)
    lg2 = _logits(x, ln_g, ln_b, tb2)
    for r in rows:
        t = int(top[r])
        assert lg2[r, t - 1] == lg2[r, t] == lg2[r, t + 1]
    assert (ranks[rows] == 2).all(), ranks[rows]       # the copy below counts, the copy above does not
    _assert_same((m, ranks), Fn.eval_rank_metrics(lg2, tg, want_ranks=True))


# ------------------------------------------------------------------------------------------------ 3. agreement with recommend
def _exclusions(lg, E, seed, targets):
    """[R, E]: each row's true top-5, random ids, duplicates, 0 and out-of-range ids, and in every 7th row the target, shuffled"""
    R, C = lg.shape
    g = torch.Generator().manual_seed(seed)
    masked = lg.clone()
    masked[:, 0] = NEG
    top = masked.topk(5, dim=1).indices.cpu()
    ex = torch.randint(1, C, (R, E), generator=g)
    junk = torch.tensor([0, -3, C, C + 7, 1 << 40])
    for r in range(R):
        fixed = torch.cat([top[r], top[r, :2], junk] + ([targets[r:r + 1].cpu()] if r % 7 == 0 else []))[:E]
        ex[r, :len(fixed)] = fixed
        ex[r] = ex[r, torch.randperm(E, generator=g)]
    return ex.cuda()


@pytest.mark.parametrize("R,D,C,E", [(200, 128, 20000, 40), (64, 64, 5000, 5000), (130, 256, 3001, 13), (129, 128, 1000001, 300)])
def test_agrees_with_recommend_under_exclusions(R, D, C, E):
    x, ln_g, ln_b, tb = _head(R, D, C, seed=C + E)
    lg = _logits(x, ln_g, ln_b, tb)
    g = torch.Generator().manual_seed(E)
    masked = lg.clone()
    masked[:, 0] = NEG
    near = masked.topk(100, dim=1).indices
    tg = near[torch.arange(R), torch.randint(0, 100, (R,), generator=g).cuda()]   # targets among each row's best 100
    ex = _exclusions(lg, E, seed=R, targets=tg)
    m, ranks = Fn.head_rank_metrics(x, ln_g, ln_b, tb, EPS, tg, exclude=ex, want_ranks=True)
    top = Fn.head_topk(x, ln_g, ln_b, tb, EPS, 64, ex)
    excluded = (ex == tg[:, None]).any(1)
    assert int(excluded.sum()) >= R // 7
    assert (ranks[excluded] == 0).all()
    keep = ~excluded
    hit = top.items == tg[:, None]
    assert torch.equal((ranks[keep] <= 64) & (ranks[keep] >= 1), hit[keep].any(1))
    rows = (keep & (ranks <= 64)).nonzero()[:, 0]
    assert len(rows) >= R // 8
    assert torch.equal(top.items[rows, ranks[rows].long() - 1], tg[rows])
    assert torch.equal(top.scores[rows, ranks[rows].long() - 1], lg[rows, tg[rows]])
    # the logits path with the excluded ids at -inf and the excluded targets dropped
    lg2 = lg.clone()
    lg2.scatter_(1, torch.where((ex >= 1) & (ex < C), ex, 0), NEG)
    tg2 = torch.where(excluded, torch.zeros_like(tg), tg)
    _assert_same((m, ranks), Fn.eval_rank_metrics(lg2, tg2, want_ranks=True))


# ------------------------------------------------------------------------------------------------ 4. models
def _hstu(D=64, H=2, use_time=True, seed=0):
    from tests.hstu_cases import _serve_model
    return _serve_model(D, H, use_time=use_time, seed=seed)


@pytest.mark.parametrize("timestamps", [True, False])
def test_hstu_evaluate_batch_matches_last_logits(timestamps):
    from tests.util import make_batch
    m = _hstu(128, 4, seed=2)
    ids, ts, _ = make_batch(40, 50, m.num_items, seed=3, device="cuda")     # includes left-padded and all-padding rows
    ts = ts if timestamps else None
    tg = _targets(40, m.num_items + 1, seed=4)
    got = m.evaluate_batch(ids, ts, tg)
    got = m.evaluate_batch(ids, ts, tg, got)                                 # accumulates
    ref = Fn.eval_rank_metrics(m.last_logits(ids, ts), tg)
    ref = Fn.eval_rank_metrics(m.last_logits(ids, ts), tg, ref)
    assert torch.equal(got[:3], ref[:3])
    torch.testing.assert_close(got[3:], ref[3:], rtol=1e-5, atol=1e-5)
    # with exclusions: the logits with the excluded ids at -inf, excluded targets not ranked
    ex = torch.randint(-2, m.num_items + 3, (40, 30), device="cuda")
    ex[::5, 0] = tg[::5]
    lg = m.last_logits(ids, ts)
    lg.scatter_(1, torch.where((ex >= 1) & (ex <= m.num_items), ex, 0), NEG)
    tg2 = torch.where((ex == tg[:, None]).any(1), torch.zeros_like(tg), tg)
    got = m.evaluate_batch(ids, ts, tg, exclude=ex)
    ref = Fn.eval_rank_metrics(lg, tg2)
    assert torch.equal(got[:3], ref[:3])
    torch.testing.assert_close(got[3:], ref[3:], rtol=1e-5, atol=1e-5)


def test_hstu_evaluate_batch_at_fp32_is_the_logits_path():
    from tests.util import make_batch
    m = _hstu(64, 2, seed=6)
    m.set_precision("fp32")
    ids, ts, _ = make_batch(9, 30, m.num_items, seed=5, device="cuda")
    tg = _targets(9, m.num_items + 1, seed=1)
    got = m.evaluate_batch(ids, ts, tg)
    assert torch.equal(got, Fn.eval_rank_metrics(m.last_logits(ids, ts), tg))
    with pytest.raises(RuntimeError, match="bf16"):
        m.evaluate_batch(ids, ts, tg, exclude=torch.zeros(9, 2, dtype=torch.int64, device="cuda"))


def _trainer_loop(logits_last, targets, top_ks=(1, 5, 10)):
    """the evaluation loop of the reference SASRec trainer, per sample on the host"""
    last = logits_last.clone()
    last[:, 0] = NEG
    top = torch.topk(last, max(top_ks), dim=-1).indices
    out = [0.0] * 6
    for i in range(last.shape[0]):
        t, preds = int(targets[i]), top[i].tolist()
        for n, k in enumerate(top_ks):
            if t in preds[:k]:
                out[n] += 1.0
                out[3 + n] += 1.0 / math.log2(preds[:k].index(t) + 2.0)
    return torch.tensor(out)


def test_sasrec_evaluate_batch_matches_forward_and_the_trainer_loop():
    from genrec_b200.sasrec import SASRec
    torch.manual_seed(0)
    V, L, B = 700, 30, 48
    m = SASRec(V, L, 64, 2, 2, 256, dropout=0.0).cuda().eval()
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(1, V + 1, (B, L), generator=g)
    ids[1, :11] = 0
    ids = ids.cuda()
    logits, _ = m(ids)
    last = logits[:, -1]
    masked = last.clone()
    masked[:, 0] = NEG
    near = masked.topk(12, dim=1).indices
    tg = near[torch.arange(B), torch.randint(0, 12, (B,), generator=g).cuda()]   # many hits at every cutoff
    tg[5] = 0
    got = m.evaluate_batch(ids, tg)
    ref = Fn.eval_rank_metrics(last, tg)
    assert torch.equal(got[:3], ref[:3])
    torch.testing.assert_close(got[3:], ref[3:], rtol=1e-5, atol=1e-5)
    top = torch.sort(masked, dim=1, descending=True).values[:, :11]
    assert (top[:, 1:] < top[:, :-1]).all()                                 # no ties among the best 11: the loop is well defined
    torch.testing.assert_close(got.cpu(), _trainer_loop(last, tg.cpu()), rtol=1e-5, atol=1e-5)
    ex = torch.randint(0, V + 2, (B, 8), device="cuda")
    m2, r2 = Fn.head_rank_metrics(m.encode(ids)[:, -1, :], m.final_norm.weight, m.final_norm.bias, Fn.cast_bf16(m.item_embedding.weight),
                                  m.final_norm.eps, tg, exclude=ex, want_ranks=True)
    assert torch.equal(m.evaluate_batch(ids, tg, exclude=ex), m2)


# ------------------------------------------------------------------------------------------------ 5. memory
def test_memory_does_not_grow_with_the_catalog():
    R, D, C = 128, 128, 1000001
    x, ln_g, ln_b, tb = _head(R, D, C, seed=11)
    tg = _targets(R, C, seed=1)
    Fn.head_rank_metrics(x, ln_g, ln_b, tb, EPS, tg)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    Fn.head_rank_metrics(x, ln_g, ln_b, tb, EPS, tg, want_ranks=True)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base < R * C * 4 // 10


# ------------------------------------------------------------------------------------------------ 6. CUDA graph
def test_hstu_evaluate_batch_cuda_graph_replay():
    from tests.util import make_batch
    m = _hstu(128, 4, seed=1)
    V, B, L = m.num_items, 16, 40
    s_ids, s_ts, _ = make_batch(B, L, V, seed=0, device="cuda")
    s_tg = torch.randint(1, V + 1, (B,), device="cuda")
    s_met = torch.zeros(6, device="cuda")
    m.evaluate_batch(s_ids, s_ts, s_tg, s_met)                              # eager call first: one-time setup off the capture
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        s_met.zero_()
        m.evaluate_batch(s_ids, s_ts, s_tg, s_met)
    gen = torch.Generator().manual_seed(3)
    for step in range(4):
        ids, ts, _ = make_batch(B, L, V, seed=10 + step, device="cuda")
        tg = torch.randint(0, V + 1, (B,), generator=gen).cuda()
        ref = m.evaluate_batch(ids, ts, tg)
        s_ids.copy_(ids)
        s_ts.copy_(ts)
        s_tg.copy_(tg)
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(s_met[:3], ref[:3]), step
        torch.testing.assert_close(s_met[3:], ref[3:], rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------ 7. determinism, custom op
def test_deterministic_and_custom_op_matches_functional():
    import genrec_b200.ops  # noqa: F401
    R, D, C = 300, 128, 50000
    x, ln_g, ln_b, tb = _head(R, D, C, seed=5)
    tg = _targets(R, C, seed=5)
    ex = torch.randint(-1, C + 2, (R, 17), device="cuda")
    m0, r0 = Fn.head_rank_metrics(x, ln_g, ln_b, tb, EPS, tg, exclude=ex, want_ranks=True)
    for _ in range(3):
        m1, r1 = Fn.head_rank_metrics(x, ln_g, ln_b, tb, EPS, tg, exclude=ex, want_ranks=True)
        assert torch.equal(r0, r1) and torch.equal(m0[:3], m1[:3])
    for e in (ex, None):
        om, orank = torch.ops.genrec_b200.head_rank_metrics(x, ln_g, ln_b, tb, EPS, tg, e)
        fm, frank = Fn.head_rank_metrics(x, ln_g, ln_b, tb, EPS, tg, exclude=e, want_ranks=True)
        assert torch.equal(orank, frank) and torch.equal(om[:3], fm[:3])
        torch.testing.assert_close(om, fm, rtol=1e-5, atol=1e-5)
