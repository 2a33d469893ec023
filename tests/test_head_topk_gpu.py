"""grb_head_topk (Fn.head_topk, HSTU.recommend, extend / extend_users with top_k, SASRec.recommend) against the logits path:
head_logits of the same rows, item 0 and the excluded ids set to -inf, a stable descending sort, the first k, and item 0 in every
slot whose score is -inf.  Scores and items must match exactly: the fused kernel accumulates every score as the logits GEMM does."""
import pytest
import torch

import genrec_b200.functional as Fn
from tests.head_cases import EPS, NEG, _assert_same, _head, _select

pytestmark = pytest.mark.gpu


def _reference(x, ln_g, ln_b, tb, eps, k, exclude=None):
    logits = Fn.head_logits(x[:, None, :], ln_g, ln_b, tb, tb, eps)[:, 0, :]
    return _select(logits, k, exclude)


def _exclusions(x, ln_g, ln_b, tb, E, seed):
    """[R, E]: each row's true top-5 ids, random ids, duplicates, 0 and out-of-range ids, shuffled"""
    R, C = x.shape[0], tb.shape[0]
    g = torch.Generator().manual_seed(seed)
    top = _reference(x, ln_g, ln_b, tb, EPS, 5)[1].cpu()
    ex = torch.randint(1, C, (R, E), generator=g)
    junk = torch.tensor([0, -3, C, C + 7, 1 << 40])
    for r in range(R):
        fixed = torch.cat([top[r], top[r, :2], junk])[:E]
        ex[r, :len(fixed)] = fixed
        ex[r] = ex[r, torch.randperm(E, generator=g)]
    return ex.cuda()


CASES = [(1, 128, 12102, 10, 0), (128, 128, 12102, 10, 50), (200, 64, 129, 64, 0), (300, 128, 50000, 17, 0), (7, 128, 1000001, 64, 100),
         (5, 256, 3001, 1, 9), (130, 64, 2, 3, 0), (1, 64, 3, 64, 0)]


@pytest.mark.parametrize("R,D,C,k,E", CASES)
def test_matches_sorted_logits(R, D, C, k, E):
    x, ln_g, ln_b, tb = _head(R, D, C, seed=R + D + C)
    ex = _exclusions(x, ln_g, ln_b, tb, E, seed=E) if E else None
    got = Fn.head_topk(x, ln_g, ln_b, tb, EPS, k, ex)
    _assert_same(got, _reference(x, ln_g, ln_b, tb, EPS, k, ex))


def test_fewer_eligible_items_than_k():
    R, D, C, k, E = 3, 256, 1000, 64, 990
    x, ln_g, ln_b, tb = _head(R, D, C, seed=5)
    g = torch.Generator().manual_seed(6)
    ex = torch.stack([torch.randperm(C - 1, generator=g)[:E] + 1 for _ in range(R)]).cuda()
    got = Fn.head_topk(x, ln_g, ln_b, tb, EPS, k, ex)
    ref = _reference(x, ln_g, ln_b, tb, EPS, k, ex)
    _assert_same(got, ref)
    assert (got.scores[:, C - 1 - E:] == NEG).all() and (got.items[:, C - 1 - E:] == 0).all()
    assert torch.isfinite(got.scores[:, :C - 1 - E]).all()


def _split_edges(R, C):
    """first item of every per-CTA item range of the kernel (the split rule of carve_sweep in api.cu)"""
    num_m, num_n = -(-R // 128), -(-C // 128)
    splits = max(1, min(torch.cuda.get_device_properties(0).multi_processor_count // num_m, num_n, 256))
    return sorted({s * num_n // splits * 128 for s in range(1, splits)})


@pytest.mark.parametrize("R,C,k", [(8, 50000, 17), (130, 300001, 64), (3, 2000, 40)])
def test_exact_ties_go_to_the_lower_id(R, C, k):
    D = 128
    x, ln_g, ln_b, tb = _head(R, D, C, seed=C)
    tb = (tb.float() * 0.01).to(torch.bfloat16)
    edges = [e for e in _split_edges(R, C) if e < C]
    ids = sorted({i for e in [128, 256] + edges for i in (e - 1, e, e + 1) if 1 <= i < C} | {1, 2, C - 1})
    half = len(ids) // 2
    g = torch.Generator().manual_seed(1)
    v = torch.randn(D, generator=g).to(torch.bfloat16).cuda()
    for j, i in enumerate(ids):             # two tied groups, +v and -v: for every row one of them holds the largest scores
        tb[i] = v if j % 2 == 0 or j < half else -v
    got = Fn.head_topk(x, ln_g, ln_b, tb, EPS, k)
    _assert_same(got, _reference(x, ln_g, ln_b, tb, EPS, k))
    # a table whose rows are all equal: items 1..k, in order
    flat = v[None, :].expand(C, D).contiguous()
    got = Fn.head_topk(x, ln_g, ln_b, flat, EPS, k)
    assert (got.items == torch.arange(1, min(k, C - 1) + 1, device="cuda")[None, :]).all()
    _assert_same(got, _reference(x, ln_g, ln_b, flat, EPS, k))


def test_deterministic():
    x, ln_g, ln_b, tb = _head(300, 128, 200001, seed=3)
    ex = _exclusions(x, ln_g, ln_b, tb, 40, seed=4)
    a = Fn.head_topk(x, ln_g, ln_b, tb, EPS, 33, ex)
    b = Fn.head_topk(x, ln_g, ln_b, tb, EPS, 33, ex)
    assert torch.equal(a.scores, b.scores) and torch.equal(a.items, b.items)


def test_custom_op_matches_functional():
    import genrec_b200.ops  # noqa: F401
    x, ln_g, ln_b, tb = _head(9, 64, 777, seed=8)
    ex = _exclusions(x, ln_g, ln_b, tb, 4, seed=2)
    s, i = torch.ops.genrec_b200.head_topk(x, ln_g, ln_b, tb, EPS, 12, ex)
    _assert_same((s, i), _reference(x, ln_g, ln_b, tb, EPS, 12, ex))


def test_memory_does_not_grow_with_the_catalog():
    B, D, C, k = 128, 128, 1000001, 64
    x, ln_g, ln_b, tb = _head(B, D, C, seed=11)
    Fn.head_topk(x, ln_g, ln_b, tb, EPS, k)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    Fn.head_topk(x, ln_g, ln_b, tb, EPS, k)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base < B * C * 4 // 8


# ------------------------------------------------------------------------------------------------ models
def _hstu(D=64, H=2, use_time=True, seed=0):
    from tests.hstu_cases import _serve_model
    return _serve_model(D, H, use_time=use_time, seed=seed)


@pytest.mark.parametrize("timestamps", [True, False])
def test_hstu_recommend_matches_last_logits(timestamps):
    from tests.util import make_batch
    m = _hstu()
    ids, ts, _ = make_batch(6, 40, m.num_items, seed=3, device="cuda")      # rows 1 (left-padded) and 2 (all padding)
    ts = ts if timestamps else None
    ex = torch.randint(-2, m.num_items + 3, (6, 30), device="cuda")
    for k, e in ((10, None), (64, ex), (1, ex[:, :0])):
        got = m.recommend(ids, ts, top_k=k, exclude=e)
        assert isinstance(got, Fn.TopItems)
        _assert_same(got, _select(m.last_logits(ids, ts), k, e))


def test_hstu_recommend_equals_predict_without_ties():
    from tests.util import make_batch
    m = _hstu(128, 4, seed=5)
    ids, ts, _ = make_batch(8, 50, m.num_items, seed=9, device="cuda")
    k = 10
    last = m.last_logits(ids, ts)
    last[:, 0] = NEG
    top = torch.sort(last, dim=1, descending=True).values[:, :k + 1]
    rows = (top[:, 1:] < top[:, :-1]).all(1)                                # rows without a tie among their top k + 1
    assert int(rows.sum()) >= 6
    assert torch.equal(m.recommend(ids, ts, top_k=k).items[rows], m.predict(ids, ts, top_k=k)[rows])


def test_sasrec_recommend_matches_forward():
    from genrec_b200.sasrec import SASRec
    torch.manual_seed(0)
    V, L = 700, 30
    m = SASRec(V, L, 64, 2, 2, 256, dropout=0.0).cuda().eval()
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(1, V + 1, (5, L), generator=g)
    ids[1, :11] = 0
    ids = ids.cuda()
    ex = torch.randint(0, V + 2, (5, 8), device="cuda")
    logits, _ = m(ids)
    for k, e in ((10, None), (33, ex)):
        _assert_same(m.recommend(ids, top_k=k, exclude=e), _select(logits[:, -1], k, e))


def test_extend_with_top_k_matches_twin_state():
    from tests.hstu_cases import _absolute_ts, _chunks
    m = _hstu(128, 4)
    B = 3
    chunks = _absolute_ts(_chunks(B, [40, 1, 1, 3, 1], seed=4))
    chunks[2][0][1] = 0                                                       # an all-pad row
    a, b = m.new_state(B, 64), m.new_state(B, 64)
    g = torch.Generator().manual_seed(0)
    for ids, ts in chunks:
        ex = torch.randint(0, m.num_items + 2, (B, 7), generator=g).cuda()
        logits = m.extend(a, ids.cuda(), ts.cuda())
        got = m.extend(b, ids.cuda(), ts.cuda(), top_k=10, exclude=ex)
        _assert_same(got, _select(logits, 10, ex))
    for x, y in zip((a.kv, a.lengths, a.last_hidden), (b.kv, b.lengths, b.last_hidden)):
        assert torch.equal(x, y)


def test_extend_users_with_top_k_matches_twin_pool():
    m = _hstu(64, 2)
    V = m.num_items
    pa, pb = (m.new_pool(max_users=6, num_pages=16, page_size=64, max_items=192) for _ in range(2))
    g = torch.Generator().manual_seed(7)
    t = [1_300_000_000]

    def chunk(B, n):
        ids = torch.randint(1, V + 1, (B, n), generator=g)
        t[0] += 10 ** 6
        return ids.cuda(), (t[0] + torch.arange(B * n).view(B, n) * 60).cuda()

    calls = [([0, 1, 2, 3], 50), ([2, 0], 1), ([5, 1, 3], 1), ("release", [1]), ([1, 4], 2), ("allpad", [0, 3]),
             (torch.tensor([2, 4, 2], device="cuda"), 1), ([3, 2, 0], 1)]
    for users, n in calls:
        if isinstance(users, str) and users == "release":
            pa.release(n)
            pb.release(n)
            continue
        allpad = isinstance(users, str) and users == "allpad"
        if allpad:
            users, n = n, 1
        B = len(users)
        ids, ts = chunk(B, n)
        if allpad:
            ids[0] = 0
        ex = torch.randint(-1, V + 2, (B, 5), generator=g).cuda()
        logits = m.extend_users(pa, users, ids, ts)
        got = m.extend_users(pb, users, ids, ts, top_k=10, exclude=ex)
        _assert_same(got, _select(logits, 10, ex))
    assert int(pb.errors()) == pb.ERR_USER_REPEAT and torch.equal(pa.last_hidden, pb.last_hidden)


def test_extend_users_top_k_cuda_graph_replay():
    from tests.hstu_cases import _fill
    m = _hstu(128, 4)
    V = m.num_items
    eager = m.new_pool(max_users=6, num_pages=16, page_size=64, max_items=192)
    graphed = m.new_pool(max_users=6, num_pages=16, page_size=64, max_items=192)
    for p in (eager, graphed):
        _fill(m, p, [0, 1, 2, 3, 4, 5], 62, seed=8)
    s_users = torch.tensor([0, 1, 2], device="cuda")
    s_ids = torch.zeros(3, 2, dtype=torch.int64, device="cuda")
    s_ts = torch.zeros(3, 2, dtype=torch.int64, device="cuda")
    s_ex = torch.zeros(3, 4, dtype=torch.int64, device="cuda")
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        out = m.extend_users(graphed, s_users, s_ids, s_ts, top_k=10, exclude=s_ex)
    gen = torch.Generator().manual_seed(3)
    t = 1_400_000_000
    for step in range(4):
        users = torch.randperm(6, generator=gen)[:3]
        ids = torch.randint(1, V + 1, (3, 2), generator=gen)
        ex = torch.randint(0, V + 1, (3, 4), generator=gen)
        ts = t + torch.arange(6).view(3, 2) * 100
        t += 1000
        ref = m.extend_users(eager, users, ids.cuda(), ts.cuda(), top_k=10, exclude=ex.cuda())
        for s, v in ((s_users, users), (s_ids, ids), (s_ts, ts), (s_ex, ex)):
            s.copy_(v)
        gr.replay()
        torch.cuda.synchronize()
        assert torch.equal(out.scores, ref.scores) and torch.equal(out.items, ref.items), step


def test_argument_errors_raise_before_any_launch():
    from genrec_b200 import _lib
    from tests.util import make_batch
    m = _hstu()
    ids, ts, _ = make_batch(3, 10, m.num_items, seed=1, device="cuda")
    st = m.new_state(3, 32)
    pool = m.new_pool(max_users=4, num_pages=4)
    m.recommend(ids, ts)
    n0 = _lib.launches()
    bad = [dict(top_k=0), dict(top_k=65), dict(top_k=2.5), dict(exclude=torch.zeros(3, dtype=torch.int64, device="cuda")),
           dict(exclude=torch.zeros(2, 4, dtype=torch.int64, device="cuda")), dict(exclude=torch.zeros(3, 4, dtype=torch.int32, device="cuda")),
           dict(exclude=torch.zeros(3, 4, dtype=torch.int64))]
    for kw in bad:
        k = kw.get("top_k", 5)
        e = kw.get("exclude")
        with pytest.raises(ValueError):
            m.recommend(ids, ts, top_k=k, exclude=e)
        with pytest.raises(ValueError):
            m.extend(st, ids, ts, top_k=k, exclude=e)
        with pytest.raises(ValueError):
            m.extend_users(pool, [0, 1, 2], ids, ts, top_k=k, exclude=e)
    with pytest.raises(ValueError, match="top_k"):
        m.extend(st, ids, ts, exclude=torch.zeros(3, 4, dtype=torch.int64, device="cuda"))
    with pytest.raises(ValueError):
        Fn.head_topk(torch.zeros(3, 64, device="cuda"), m.final_norm.weight, m.final_norm.bias, m._table_mirror(), EPS, 0)
    m.set_precision("fp32")
    with pytest.raises(RuntimeError, match="bf16"):
        m.recommend(ids, ts)
    with pytest.raises(RuntimeError, match="bf16"):
        m.extend(st, ids, ts, top_k=5)
    assert _lib.launches() == n0
    assert int(st.lengths.sum()) == 0 and int(pool.lengths.sum()) == 0
