"""The paged serving pool (HSTU.new_pool / HSTU.extend_users / HSTUPool.release): bit-identical to the dense HSTUState on the same
users, arbitrary user subsets against the fp64 oracle, release and reuse, page exhaustion, refusals, determinism and CUDA graphs."""
import pytest
import torch

from tests.sign_fixed_buckets import use_sign_fixed_oracle
from tests.hstu_cases import (SERVE_V as V, _absolute_ts, _check_extend as _check, _chunks, _fill, _history_calls, _left_padded,
                              _serve_model as _model, _sign_fixed)

pytestmark = pytest.mark.gpu

WIDTHS = [1, 7, 64, 65, 63]


def _gather(pool, u):
    """user u's cached K | V rows [num_blocks, len, 2D] and timestamps [len], read through the page table"""
    L = int(pool.lengths[u])
    pages = pool.page_table[u, :-(-L // pool.page_size)].long()
    kv = pool.kv[:, pages].reshape(pool.kv.shape[0], -1, pool.kv.shape[-1])[:, :L]
    return kv, pool.timestamps[pages].reshape(-1)[:L]


def _pool_tensors(pool):
    return [pool.kv, pool.timestamps, pool.page_table, pool.lengths, pool.overflow, pool.free_stack, pool.free_top, pool.error_bits,
            pool.last_hidden]


def _same_user(pool, u, st, b):
    kv, ts = _gather(pool, u)
    L = int(st.lengths[b])
    assert int(pool.lengths[u]) == L
    assert torch.equal(kv, st.kv[:, b, :L]) and torch.equal(ts, st.timestamps[b, :L])
    assert torch.equal(pool.last_hidden[u], st.last_hidden[b])


@pytest.mark.parametrize("D,H", [(64, 2), (128, 4), (256, 8)])
@pytest.mark.parametrize("use_time", [True, False])
@pytest.mark.parametrize("order", ["rows", "permuted", "interleaved"])
def test_bit_identical_to_dense_state(D, H, use_time, order):
    m = _model(D, H, use_time=use_time)
    B, cap = 3, sum(WIDTHS)
    chunks = _absolute_ts(_chunks(B, WIDTHS, seed=D + H))
    st = m.new_state(B, cap)
    pool = m.new_pool(max_users=8, num_pages=20, page_size=64, max_items=cap)
    user_of = torch.arange(B) if order == "rows" else torch.tensor([5, 0, 3])
    if order == "interleaved":                    # scramble the free stack and keep a foreign user's pages between ours
        _fill(m, pool, [1, 6, 2], 70, seed=1)
        pool.release([6, 1])
    g = torch.Generator().manual_seed(D)
    for k, (ids, ts) in enumerate(chunks):
        ref = m.extend(st, ids.cuda(), ts.cuda())
        perm = torch.arange(B) if order == "rows" else torch.randperm(B, generator=g)
        out = m.extend_users(pool, user_of[perm], ids[perm].cuda(), ts[perm].cuda())
        assert torch.equal(out, ref[perm.cuda()]), (k, (out - ref[perm.cuda()]).abs().max())
    for b in range(B):
        _same_user(pool, int(user_of[b]), st, b)
    assert not pool.overflowed().any() and int(pool.errors()) == 0


@pytest.mark.parametrize("buckets", ["reference", "sign_fixed"])
def test_arbitrary_subsets_match_full_forward(buckets, monkeypatch):
    m = _model(64, 2, seed=3)
    if buckets == "sign_fixed":
        _sign_fixed(m)
        use_sign_fixed_oracle(monkeypatch)
        assert not m.layers[0].position_bias.uniform_of(192, "cuda")[0]
    nusers = 8
    pool = m.new_pool(max_users=nusers, num_pages=3 * nusers, page_size=64, max_items=192)   # 20 chunks of <= 9 slots fit
    hist = {u: ([], []) for u in range(nusers)}
    prev = {}
    for users, ids, ts in _history_calls(nusers, 20, seed=17):
        out = m.extend_users(pool, users, ids.cuda(), ts.cuda())
        for r, u in enumerate(users.tolist()):
            keep = ids[r] != 0
            hist[u][0].extend(ids[r][keep].tolist())
            hist[u][1].extend(ts[r][keep].tolist())
            if not keep.any() and u in prev:
                assert torch.equal(out[r], prev[u])            # an all-pad row keeps its user's logits
            prev[u] = out[r].clone()
        rows = [r for r, u in enumerate(users.tolist()) if hist[u][0]]
        if rows:
            cids, cts = _left_padded(hist, users)
            _check(out, m, cids.cuda(), cts.cuda(), rows)
    assert pool.lengths.tolist() == [len(hist[u][0]) for u in range(nusers)]
    assert not pool.overflowed().any() and int(pool.errors()) == 0


def test_release_and_reuse():
    m = _model(128, 4)
    pool = m.new_pool(max_users=6, num_pages=12, page_size=64, max_items=192)
    _fill(m, pool, [0, 1, 2, 3], 100, seed=2)
    assert int(pool.pages_free()) == 12 - 8
    chunks = _absolute_ts(_chunks(1, [5, 70, 3], seed=9))
    pool.release([1])
    assert int(pool.pages_free()) == 12 - 6 and int(pool.lengths[1]) == 0 and not pool.last_hidden[1].any()
    fresh = m.new_pool(max_users=6, num_pages=12, page_size=64, max_items=192)
    for ids, ts in chunks:                                     # the refilled slot computes what a fresh pool computes
        a = m.extend_users(pool, [1], ids.cuda(), ts.cuda())
        b = m.extend_users(fresh, [1], ids.cuda(), ts.cuda())
        assert torch.equal(a, b)
    for x, y in zip(_gather(pool, 1), _gather(fresh, 1)):
        assert torch.equal(x, y)
    assert torch.equal(pool.last_hidden[1], fresh.last_hidden[1])
    pool.release(torch.tensor([3, 0, 2, 1], device="cuda"))    # device users: no host checks, same effect
    assert int(pool.pages_free()) == 12
    assert sorted(pool.free_stack.tolist()) == list(range(12))
    assert not pool.lengths.any() and not pool.last_hidden.any() and int(pool.errors()) == 0


def test_exhaustion_drops_in_row_order():
    m = _model(64, 2)
    g = torch.Generator().manual_seed(4)
    ids = torch.randint(1, V + 1, (3, 100), generator=g).cuda()
    ts = (1_300_000_000 + torch.cumsum(torch.randint(1, 86400, (3, 100), generator=g), 1)).cuda()
    big = m.new_pool(max_users=4, num_pages=10, page_size=64, max_items=192)
    ref = m.extend_users(big, torch.tensor([0, 1, 2], device="cuda"), ids, ts)
    for rows, short in (([0, 1, 2], 2), ([2, 0, 1], 1)):     # 6 pages wanted, 5 free: the last row gets one page
        small = m.new_pool(max_users=4, num_pages=5, page_size=64, max_items=192)
        r = torch.tensor(rows, device="cuda")
        out = m.extend_users(small, r, ids[r], ts[r])          # device users: the host page check is skipped
        assert small.lengths.tolist()[:3] == [64 if u == short else 100 for u in range(3)]
        assert small.overflowed().tolist()[:3] == [u == short for u in range(3)]
        assert int(small.pages_free()) == 0
        for k, u in enumerate(rows):                           # users that found their pages are as in a pool with room
            if u != short:
                assert torch.equal(out[k], ref[u])
                for x, y in zip(_gather(small, u), _gather(big, u)):
                    assert torch.equal(x, y)
    # max_items: 100 + 100 > 192 -> user 0 keeps 192 items and is flagged; user 1 (all padding) is untouched
    more = ids[:2].clone()
    more_ts = ts[:2] + 10 ** 7
    more[1] = 0
    m.extend_users(big, torch.tensor([0, 1], device="cuda"), more, more_ts)
    assert big.lengths.tolist()[:3] == [192, 100, 100] and big.overflowed().tolist()[:3] == [True, False, False]


def test_refusals():
    from genrec_b200 import _lib
    m = _model(64, 2)
    pool = m.new_pool(max_users=4, num_pages=3, page_size=64, max_items=128)
    ids = torch.randint(1, V + 1, (2, 80), device="cuda")
    ts = 1_300_000_000 + torch.cumsum(torch.randint(1, 86400, (2, 80), device="cuda"), 1)
    m.extend_users(pool, [0, 1], ids[:, :60], ts[:, :60])    # host bounds: 60 items and one page per user
    n0 = _lib.launches()
    for users, n, match in (([0, 0], 1, "distinct"), ([0, 4], 1, "range"), ([-1, 1], 1, "range"), ([0, 1], 70, "max_items"),
                            ([2, 3], 60, "pages")):
        with pytest.raises(ValueError, match=match):
            m.extend_users(pool, users, ids[:, :n], ts[:, :n])
        assert _lib.launches() == n0, match                   # refused before any launch
    with pytest.raises(ValueError, match="distinct"):
        pool.release([1, 1])
    with pytest.raises(ValueError, match="timestamps"):
        m.extend_users(pool, [0, 1], ids[:, :1], None)
    assert _lib.launches() == n0
    for p in m.parameters():                                  # stale pool: a torch optimizer step
        p.grad = torch.ones_like(p)
    torch.optim.Adam(m.parameters(), lr=1e-3).step()
    with pytest.raises(RuntimeError, match="rebuild"):
        m.extend_users(pool, [0], ids[:1, :1], ts[:1, :1])
    md = _model(64, 2, dropout=0.2).train()
    with pytest.raises(RuntimeError, match="dropout"):
        md.extend_users(md.new_pool(4, 4), [0], ids[:1], ts[:1])
    m.set_precision("fp32")
    with pytest.raises(RuntimeError, match="bf16"):
        m.extend_users(m.new_pool(4, 4), [0], ids[:1], ts[:1])
    assert _lib.launches() == n0


def test_device_users_duplicate_and_range_set_errors():
    m = _model(64, 2)
    pool = m.new_pool(max_users=4, num_pages=8, page_size=64, max_items=128)
    ids = torch.randint(1, V + 1, (3, 5), device="cuda")
    ts = 1_300_000_000 + torch.cumsum(torch.randint(1, 86400, (3, 5), device="cuda"), 1)
    out = m.extend_users(pool, torch.tensor([2, 1, 2], device="cuda"), ids, ts)
    assert int(pool.errors()) == pool.ERR_USER_REPEAT
    assert pool.lengths.tolist() == [0, 5, 5, 0]              # the repeated row counts as padding
    ref = m.new_pool(max_users=4, num_pages=8, page_size=64, max_items=128)
    r = m.extend_users(ref, torch.tensor([2, 1, 3], device="cuda"), ids[:, :5] * torch.tensor([[1], [1], [0]], device="cuda"), ts)
    assert torch.equal(out[:2], r[:2]) and torch.equal(out[2], r[2])   # the rejected row gets the head of a zero vector
    m.extend_users(pool, torch.tensor([7, 0], device="cuda"), ids[:2], ts[:2] + 10 ** 6)
    assert int(pool.errors()) == pool.ERR_USER_REPEAT | pool.ERR_USER_RANGE
    assert pool.lengths.tolist() == [5, 5, 5, 0]


def test_deterministic():
    m = _model(128, 4)
    runs = []
    for _ in range(2):
        pool = m.new_pool(max_users=8, num_pages=40, page_size=64, max_items=384)
        outs = [m.extend_users(pool, users, ids.cuda(), ts.cuda()) for users, ids, ts in _history_calls(8, 12, seed=5)]
        _fill(m, pool, [6, 2, 5], 150, seed=6)
        runs.append((outs, [t.clone() for t in _pool_tensors(pool)]))
    for a, b in zip(runs[0][0], runs[1][0]):
        assert torch.equal(a, b)
    for a, b in zip(runs[0][1], runs[1][1]):
        assert torch.equal(a, b)


def test_cuda_graph_replay_with_rewritten_users():
    m = _model(128, 4)
    eager = m.new_pool(max_users=6, num_pages=16, page_size=64, max_items=192)
    graphed = m.new_pool(max_users=6, num_pages=16, page_size=64, max_items=192)
    for p in (eager, graphed):
        _fill(m, p, [0, 1, 2, 3, 4, 5], 62, seed=8)
    s_users = torch.tensor([0, 1, 2], device="cuda")
    s_ids = torch.zeros(3, 2, dtype=torch.int64, device="cuda")
    s_ts = torch.zeros(3, 2, dtype=torch.int64, device="cuda")
    s_rel = torch.tensor([0], device="cuda")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = m.extend_users(graphed, s_users, s_ids, s_ts)
    g_rel = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g_rel):
        graphed.release(s_rel)
    gen = torch.Generator().manual_seed(3)
    t = 1_400_000_000
    for step in range(6):
        users = torch.randperm(6, generator=gen)[:3]
        ids = torch.randint(1, V + 1, (3, 2), generator=gen)
        ids[step % 3, 0] = 0
        ts = t + torch.arange(6).view(3, 2) * 100
        t += 1000
        ref = m.extend_users(eager, users, ids.cuda(), ts.cuda())
        s_users.copy_(users)
        s_ids.copy_(ids)
        s_ts.copy_(ts)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, ref), step
        if step % 2:                                           # release a user, then keep extending it from scratch
            rel = users[:1]
            eager.release(rel)
            s_rel.copy_(rel)
            g_rel.replay()
        for a, b in zip(_pool_tensors(graphed), _pool_tensors(eager)):
            assert torch.equal(a, b), step
