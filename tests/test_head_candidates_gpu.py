"""grb_head_candidates (Fn.head_candidates, HSTU.retrieve, SASRec.retrieve, extend / extend_users with num_candidates) against the
logits path: head_logits of the same rows, item 0 and the excluded ids set to -inf, a stable descending sort, the first k, and item
0 in every slot whose score is -inf (the rule of test_head_topk_gpu.py).  Scores and items must match exactly."""
import pytest
import torch

import genrec_b200.functional as Fn
from tests.head_cases import EPS, NEG, _assert_same, _head, _select

pytestmark = pytest.mark.gpu


def _reference(x, ln_g, ln_b, tb, eps, k, exclude=None, chunk=128):
    """_select of head_logits, a row chunk at a time (the [R, C] logits of R = 1,024 rows at C = 1,000,001 would take 4 GB)"""
    out = []
    for r0 in range(0, x.shape[0], chunk):
        logits = Fn.head_logits(x[r0:r0 + chunk, None, :], ln_g, ln_b, tb, tb, eps)[:, 0, :]
        out.append(_select(logits, k, exclude[r0:r0 + chunk] if exclude is not None else None))
        del logits
    return torch.cat([s for s, _ in out]), torch.cat([i for _, i in out])


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


CASES = [(1, 128, 1000001, 2048, 0), (7, 64, 1000001, 500, 100), (128, 128, 1000001, 1024, 0), (130, 256, 1000001, 65, 40),
         (1024, 128, 1000001, 2048, 0), (1024, 64, 12102, 2048, 30), (1024, 256, 3001, 500, 0), (130, 256, 12102, 2048, 50),
         (128, 64, 12102, 65, 0), (7, 256, 3001, 2048, 9), (128, 128, 3001, 1, 0), (7, 128, 129, 500, 0), (1, 64, 129, 65, 3),
         (130, 64, 2, 500, 0), (1, 256, 2, 1, 0), (128, 128, 12102, 64, 30), (7, 64, 3001, 64, 0)]


@pytest.mark.parametrize("R,D,C,k,E", CASES)
def test_matches_sorted_logits(R, D, C, k, E):
    x, ln_g, ln_b, tb = _head(R, D, C, seed=R + D + C + k)
    ex = _exclusions(x, ln_g, ln_b, tb, E, seed=E) if E else None
    got = Fn.head_candidates(x, ln_g, ln_b, tb, EPS, k, ex)
    assert isinstance(got, Fn.TopItems) and got.scores.shape == (R, k) and got.items.shape == (R, k)
    _assert_same(got, _reference(x, ln_g, ln_b, tb, EPS, k, ex))


def test_fewer_eligible_items_than_k():
    R, D, C, k, E = 3, 128, 3000, 2048, 2000
    x, ln_g, ln_b, tb = _head(R, D, C, seed=5)
    g = torch.Generator().manual_seed(6)
    ex = torch.stack([torch.randperm(C - 1, generator=g)[:E] + 1 for _ in range(R)]).cuda()
    got = Fn.head_candidates(x, ln_g, ln_b, tb, EPS, k, ex)
    _assert_same(got, _reference(x, ln_g, ln_b, tb, EPS, k, ex))
    n = C - 1 - E
    assert (got.scores[:, n:] == NEG).all() and (got.items[:, n:] == 0).all()
    assert torch.isfinite(got.scores[:, :n]).all()


def _split_edges(R, C, k):
    """first item of every per-CTA item range of the sweeps (carve_sweep and carve_cand in api.cu)"""
    num_m, num_n = -(-R // 128), -(-C // 128)
    splits = max(1, min(torch.cuda.get_device_properties(0).multi_processor_count // num_m, num_n, 256))
    splits = max(splits, min(-(-2 * k // 32), num_n))
    return sorted({s * num_n // splits * 128 for s in range(1, splits)})


@pytest.mark.parametrize("R,C,k", [(8, 50000, 500), (130, 300001, 2048), (3, 5000, 1000)])
def test_exact_ties_go_to_the_lower_id(R, C, k):
    D = 128
    x, ln_g, ln_b, tb = _head(R, D, C, seed=C)
    tb = (tb.float() * 0.01).to(torch.bfloat16)
    edges = [e for e in _split_edges(R, C, k) if e < C]
    ids = sorted({i for e in [128, 256] + edges for i in (e - 1, e, e + 1) if 1 <= i < C} | {1, 2, C - 1})
    half = len(ids) // 2
    g = torch.Generator().manual_seed(1)
    v = torch.randn(D, generator=g).to(torch.bfloat16).cuda()
    for j, i in enumerate(ids):             # two tied groups, +v and -v: for every row one of them holds the largest scores
        tb[i] = v if j % 2 == 0 or j < half else -v
    _assert_same(Fn.head_candidates(x, ln_g, ln_b, tb, EPS, k), _reference(x, ln_g, ln_b, tb, EPS, k))


def test_flat_table_overflows_and_stays_exact():
    """Every score equal: the answer is items 1..k in order, and every row's collect buffer overflows into the radix passes."""
    R, D, C, k = 5, 128, 1000001, 2048
    x, ln_g, ln_b, _ = _head(R, D, 2, seed=9)
    v = torch.randn(D, generator=torch.Generator().manual_seed(2)).to(torch.bfloat16).cuda()
    flat = v[None, :].expand(C, D).contiguous()
    got = Fn.head_candidates(x, ln_g, ln_b, flat, EPS, k)
    assert (got.items == torch.arange(1, k + 1, device="cuda")[None, :]).all()
    _assert_same(got, _reference(x, ln_g, ln_b, flat, EPS, k))
    # with exclusions: the lowest ids are taken out, so the answer starts later
    ex = torch.arange(1, 101, device="cuda").repeat(R, 1)
    ex[1] += 5000
    got = Fn.head_candidates(x, ln_g, ln_b, flat, EPS, k, ex)
    _assert_same(got, _reference(x, ln_g, ln_b, flat, EPS, k, ex))


def _clustered(R, D, C, lo, n, seed):
    """A table whose rows lo .. lo + n - 1 score above every other item for every row of x."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R, D, generator=g).cuda()
    ln_g = torch.full((D,), 0.1).cuda()
    b = torch.randn(D, generator=g)
    ln_b = b.cuda()
    tb = 0.05 * torch.randn(C, D, generator=g)
    tb[lo:lo + n] += 0.05 * b
    return x, ln_g, ln_b, tb.to(torch.bfloat16).cuda()


@pytest.mark.parametrize("R,k", [(128, 500), (128, 2048), (7, 1024)])
def test_clustered_top_items_in_one_range(R, k):
    D, C, n = 128, 1000001, 3000
    edges = _split_edges(R, C, k)
    lo = next(e for e, e2 in zip(edges, edges[1:]) if e2 - e >= n)
    x, ln_g, ln_b, tb = _clustered(R, D, C, lo, n, seed=k)
    ref = _reference(x, ln_g, ln_b, tb, EPS, n)
    assert ((ref[1] >= lo) & (ref[1] < lo + n)).all()        # the construction holds: every row's top 3,000 are the cluster
    got = Fn.head_candidates(x, ln_g, ln_b, tb, EPS, k)
    _assert_same(got, (ref[0][:, :k], ref[1][:, :k]))


def test_deterministic():
    x, ln_g, ln_b, tb = _head(300, 128, 200001, seed=3)
    ex = _exclusions(x, ln_g, ln_b, tb, 40, seed=4)
    for k in (700, 2048):
        a = Fn.head_candidates(x, ln_g, ln_b, tb, EPS, k, ex)
        b = Fn.head_candidates(x, ln_g, ln_b, tb, EPS, k, ex)
        assert torch.equal(a.scores, b.scores) and torch.equal(a.items, b.items)
        assert torch.equal(a.scores.view(torch.int32), b.scores.view(torch.int32))


@pytest.mark.parametrize("k", [1, 17, 64])
def test_small_k_gives_the_bits_of_head_topk(k):
    x, ln_g, ln_b, tb = _head(130, 128, 100001, seed=k)
    ex = _exclusions(x, ln_g, ln_b, tb, 20, seed=k)
    for e in (None, ex):
        a = Fn.head_candidates(x, ln_g, ln_b, tb, EPS, k, e)
        b = Fn.head_topk(x, ln_g, ln_b, tb, EPS, k, e)
        assert torch.equal(a.scores.view(torch.int32), b.scores.view(torch.int32)) and torch.equal(a.items, b.items)


def test_custom_op_matches_functional():
    import genrec_b200.ops  # noqa: F401
    x, ln_g, ln_b, tb = _head(9, 64, 7777, seed=8)
    ex = _exclusions(x, ln_g, ln_b, tb, 4, seed=2)
    s, i = torch.ops.genrec_b200.head_candidates(x, ln_g, ln_b, tb, EPS, 300, ex)
    _assert_same((s, i), _reference(x, ln_g, ln_b, tb, EPS, 300, ex))


def test_memory_does_not_grow_with_the_catalog():
    B, D, C, k = 128, 128, 1000001, 2048
    x, ln_g, ln_b, tb = _head(B, D, C, seed=11)
    Fn.head_candidates(x, ln_g, ln_b, tb, EPS, k)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    Fn.head_candidates(x, ln_g, ln_b, tb, EPS, k)
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base < B * C * 4 // 16


# ------------------------------------------------------------------------------------------------ models
def _hstu(D=64, H=2, use_time=True, seed=0):
    from tests.hstu_cases import _serve_model
    return _serve_model(D, H, use_time=use_time, seed=seed)


@pytest.mark.parametrize("timestamps", [True, False])
def test_hstu_retrieve_matches_last_logits(timestamps):
    from tests.util import make_batch
    m = _hstu()
    ids, ts, _ = make_batch(6, 40, m.num_items, seed=3, device="cuda")      # rows 1 (left-padded) and 2 (all padding)
    ts = ts if timestamps else None
    ex = torch.randint(-2, m.num_items + 3, (6, 30), device="cuda")
    last = m.last_logits(ids, ts)
    for k, e in ((65, None), (300, ex), (2048, ex[:, :0]), (m.num_items, ex)):
        got = m.retrieve(ids, ts, num_candidates=k, exclude=e)
        assert isinstance(got, Fn.TopItems)
        _assert_same(got, _select(last, k, e))


def test_sasrec_retrieve_matches_forward():
    from genrec_b200.sasrec import SASRec
    torch.manual_seed(0)
    V, L = 3000, 30
    m = SASRec(V, L, 64, 2, 2, 256, dropout=0.0).cuda().eval()
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(1, V + 1, (5, L), generator=g)
    ids[1, :11] = 0
    ids = ids.cuda()
    ex = torch.randint(0, V + 2, (5, 8), device="cuda")
    logits, _ = m(ids)
    for k, e in ((500, None), (2048, ex), (10, ex)):
        _assert_same(m.retrieve(ids, num_candidates=k, exclude=e), _select(logits[:, -1], k, e))


def test_extend_with_num_candidates_matches_twin_state():
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
        got = m.extend(b, ids.cuda(), ts.cuda(), num_candidates=500, exclude=ex)
        _assert_same(got, _select(logits, 500, ex))
    for x, y in zip((a.kv, a.lengths, a.last_hidden), (b.kv, b.lengths, b.last_hidden)):
        assert torch.equal(x, y)


def test_extend_users_with_num_candidates_matches_twin_pool():
    m = _hstu(64, 2)
    V = m.num_items
    pa, pb = (m.new_pool(max_users=6, num_pages=16, page_size=64, max_items=192) for _ in range(2))
    g = torch.Generator().manual_seed(7)
    t = [1_300_000_000]

    def chunk(B, n):
        ids = torch.randint(1, V + 1, (B, n), generator=g)
        t[0] += 10 ** 6
        return ids.cuda(), (t[0] + torch.arange(B * n).view(B, n) * 60).cuda()

    for users, n in (([0, 1, 2, 3], 50), ([2, 0], 1), ([5, 1, 3], 1), ([3, 2, 0], 2)):
        ids, ts = chunk(len(users), n)
        ex = torch.randint(-1, V + 2, (len(users), 5), generator=g).cuda()
        logits = m.extend_users(pa, users, ids, ts)
        got = m.extend_users(pb, users, ids, ts, num_candidates=500, exclude=ex)
        _assert_same(got, _select(logits, 500, ex))
    assert torch.equal(pa.last_hidden, pb.last_hidden)


def test_extend_users_num_candidates_cuda_graph_replay():
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
        out = m.extend_users(graphed, s_users, s_ids, s_ts, num_candidates=500, exclude=s_ex)
    gen = torch.Generator().manual_seed(3)
    t = 1_400_000_000
    for step in range(4):
        users = torch.randperm(6, generator=gen)[:3]
        ids = torch.randint(1, V + 1, (3, 2), generator=gen)
        ex = torch.randint(0, V + 1, (3, 4), generator=gen)
        ts = t + torch.arange(6).view(3, 2) * 100
        t += 1000
        ref = m.extend_users(eager, users, ids.cuda(), ts.cuda(), num_candidates=500, exclude=ex.cuda())
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
    m.retrieve(ids, ts, num_candidates=100)
    n0 = _lib.launches()
    ex = torch.zeros(3, 4, dtype=torch.int64, device="cuda")
    for kw in (dict(num_candidates=0), dict(num_candidates=2049), dict(num_candidates=2.5), dict(num_candidates=500, top_k=10),
               dict(num_candidates=500, exclude=torch.zeros(2, 4, dtype=torch.int64, device="cuda")),
               dict(num_candidates=500, exclude=torch.zeros(3, 4, dtype=torch.int64))):
        with pytest.raises(ValueError):
            m.extend(st, ids, ts, **kw)
        with pytest.raises(ValueError):
            m.extend_users(pool, [0, 1, 2], ids, ts, **kw)
        if "top_k" not in kw:
            with pytest.raises(ValueError):
                m.retrieve(ids, ts, **kw)
    with pytest.raises(ValueError, match="top_k"):
        m.extend(st, ids, ts, exclude=ex)
    with pytest.raises(ValueError):
        Fn.head_candidates(torch.zeros(3, 64, device="cuda"), m.final_norm.weight, m.final_norm.bias, m._table_mirror(), EPS, 2049)
    m.set_precision("fp32")
    with pytest.raises(RuntimeError, match="bf16"):
        m.retrieve(ids, ts)
    with pytest.raises(RuntimeError, match="bf16"):
        m.extend(st, ids, ts, num_candidates=500)
    assert _lib.launches() == n0
    assert int(st.lengths.sum()) == 0 and int(pool.lengths.sum()) == 0
