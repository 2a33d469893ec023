"""Packed (jagged) chunks for the cached extend: HSTU.extend_jagged / extend_users_jagged against the padded extend / extend_users
of the same items, bit for bit (outputs, cache bytes, page bookkeeping), the packed chunk attention against the fp64 reference
of tests/extend_reference.py, prefills against the full forward with a non-uniform position-bucket table, idle rows, the
device rules of the pool, CUDA-graph replays, and recommend_jagged / retrieve_jagged of HSTU and SASRec."""
import pytest
import torch

from tests import dense_reference as dr
from tests import extend_jagged_reference as jr
from tests import extend_reference as er
from tests.sign_fixed_buckets import use_sign_fixed_oracle
from tests.hstu_cases import SERVE_V as V, _check_extend as _check, _serve_model as _model, _sign_fixed
from tests.util import relerr

pytestmark = pytest.mark.gpu

DEV = "cuda"
EDGE = [0, 1, 63, 64, 65]
PACKED_VS_PADDED_TOL = 2e-2      # the packed-vs-padded tolerance of test_hstu_jagged_gpu.py / test_sasrec_jagged_gpu.py


# ---------------------------------------------------------------------------------------------------------------- chunks
class Users:
    """Each user's next items: random ids with a few 0 (pads) inside, timestamps increasing per user over all chunks."""

    def __init__(self, B, seed):
        self.g = torch.Generator().manual_seed(seed)
        self.last = torch.full((B,), 1_300_000_000, dtype=torch.int64)

    def chunk(self, lens, zero_frac=0.1):
        items, stamps = [], []
        for b, n in enumerate(lens):
            ids = torch.randint(1, V + 1, (n,), generator=self.g)
            ids[torch.rand(n, generator=self.g) < zero_frac] = 0
            ts = int(self.last[b]) + torch.cumsum(torch.randint(1, 10 ** 5, (n,), generator=self.g), 0)
            if n:
                self.last[b] = ts.max()
            items.append(ids)
            stamps.append(ts)
        return items, stamps


def packed(items, stamps, idle=0, seed=0, offsets_on=DEV):
    """input_ids / timestamps [T] on the device, offsets [B+1] (on offsets_on); `idle` junk rows after the sequences."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.cat(items + [torch.randint(1, V + 1, (idle,), generator=g)])
    ts = torch.cat(stamps + [torch.randint(1, 2 ** 40, (idle,), generator=g)])
    off = torch.zeros(len(items) + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(torch.tensor([len(i) for i in items], dtype=torch.int64), 0)
    return ids.to(DEV), ts.to(DEV), off.to(offsets_on)


def padded(items, stamps, n):
    """the left-padded [B, n] chunk of the same items"""
    ids = torch.zeros(len(items), n, dtype=torch.int64)
    ts = torch.zeros(len(items), n, dtype=torch.int64)
    for b, (i, t) in enumerate(zip(items, stamps)):
        if len(i):
            ids[b, n - len(i):] = i
            ts[b, n - len(i):] = t
    return ids.to(DEV), ts.to(DEV)


def state_tensors(st):
    return [st.kv, st.timestamps, st.lengths, st.overflow, st.last_hidden]


def pool_tensors(p):
    return [p.kv, p.timestamps, p.page_table, p.lengths, p.overflow, p.free_stack, p.free_top, p.error_bits, p.last_hidden]


def assert_same(a, b, what=""):
    if isinstance(a, tuple):
        for x, y in zip(a, b):
            assert torch.equal(x, y), what
    else:
        assert torch.equal(a, b), what


# ---------------------------------------------------------------------------------------------------------------- contract 1
@pytest.mark.parametrize("D,H", [(64, 2), (128, 4), (128, 2), (256, 4)])   # head dims 32, 32, 64, 64
@pytest.mark.parametrize("with_ts", [True, False])
@pytest.mark.parametrize("buckets", ["uniform", "non_uniform"])
def test_dense_state_packed_equals_padded(D, H, with_ts, buckets):
    """A prefill with lengths 0, 1, 63, 64, 65 and max_len, then packed and padded extends in turn on one state and padded ones
    on another: every call returns the same bits and the two states end equal, byte for byte."""
    m = _model(D, H)
    if buckets == "non_uniform":
        _sign_fixed(m)
    steps = [EDGE + [70], [3, 0, 1, 5, 2, 0], [1] * 6, [70, 10, 0, 64, 65, 7]]
    B, cap = 6, 300
    mixed, ref = m.new_state(B, cap), m.new_state(B, cap)
    users = Users(B, seed=D + H)
    for k, lens in enumerate(steps):
        items, stamps = users.chunk(lens)
        n = max(lens)
        pi, pt = padded(items, stamps, n)
        want = m.extend(ref, pi, pt if with_ts else None)
        if k % 2 == 0:
            ids, ts, off = packed(items, stamps, idle=5 * k, seed=k, offsets_on="cpu" if k == 2 else DEV)
            got = m.extend_jagged(mixed, ids, off, n, ts if with_ts else None)
        else:
            got = m.extend(mixed, pi, pt if with_ts else None)
        assert_same(got, want, k)
    for a, b in zip(state_tensors(mixed), state_tensors(ref)):
        assert torch.equal(a, b)


@pytest.mark.parametrize("D,H", [(64, 2), (128, 2), (256, 8)])
def test_pool_packed_equals_padded(D, H):
    """extend_users_jagged against extend_users on twin pools: subsets of users in any order, lengths 0 / 1 / 63 / 64 / 65 /
    max_len, page-crossing histories, device and CPU users and offsets; outputs, cache bytes, page tables, free stacks, errors."""
    m = _model(D, H)
    a, b = (m.new_pool(max_users=10, num_pages=40, page_size=64, max_items=320) for _ in range(2))
    users = Users(10, seed=D)
    plan = [([3, 0, 7, 9, 1, 5], EDGE + [100], "cuda"), ([9, 2, 3], [2, 0, 64], "cpu"), ([5, 4, 8, 0], [65, 1, 0, 3], "cuda"),
            ([1, 3, 7], [100, 63, 70], "cpu")]
    for k, (us, lens, where) in enumerate(plan):
        all_lens = [0] * 10
        for u, n in zip(us, lens):
            all_lens[u] = n
        items, stamps = users.chunk(all_lens)
        items, stamps = [items[u] for u in us], [stamps[u] for u in us]
        n = max(lens)
        u = torch.tensor(us, device=where)
        pi, pt = padded(items, stamps, n)
        want = m.extend_users(b, u, pi, pt, top_k=10 if k == 1 else None)
        ids, ts, off = packed(items, stamps, idle=3, seed=k, offsets_on=where)
        got = m.extend_users_jagged(a, u, ids, off, n, ts, top_k=10 if k == 1 else None)
        assert_same(got, want, k)
        for x, y in zip(pool_tensors(a), pool_tensors(b)):
            assert torch.equal(x, y), k
    assert a.pages_bound <= b.pages_bound            # CPU offsets: the exact lengths, not the chunk width
    assert int(a.error_bits) == 0


def test_append_kernels_match_the_restatement():
    """grb_hstu_cache_append_jagged / grb_hstu_pool_append_jagged against tests/extend_jagged_reference.py, with idle rows,
    empty sequences, ids 0 inside sequences, rooms that drop items, and a malformed device offsets that the kernels clamp."""
    import genrec_b200.functional as Fn
    m = _model(64, 2)
    g = torch.Generator().manual_seed(5)
    st = m.new_state(7, 80)
    st.lengths.copy_(torch.tensor([0, 5, 79, 16, 40, 1, 0], dtype=torch.int32))
    ids, ts, off = jr.random_packed_chunk(g, 7, 66, V, idle=9, lengths=[0, 66, 3, 65, 64, 1, 40])
    L0, ov0 = st.lengths.cpu(), st.overflow.cpu()
    pos, last = Fn.hstu_cache_append(st._struct(), ids.to(DEV), ts.to(DEV), off.to(DEV), 66)
    want = jr.padded_equivalent(ids, ts, off, 66, None, None, L0, ov0, 80)
    assert torch.equal(pos.cpu(), want["positions"]) and torch.equal(last.cpu(), want["last_row"])
    assert torch.equal(st.lengths.cpu(), want["lengths"]) and torch.equal(st.overflow.cpu(), want["overflow"])
    for u, q, t in want["writes"]:
        assert int(st.timestamps[u, q]) == t
    # a malformed device offsets: sequences are clamped to [0, T) and to max_len, as seq_span does
    st2 = m.new_state(4, 80)
    bad = torch.tensor([0, 30, 20, 500, 600], dtype=torch.int64)
    ids2, ts2 = ids[:50], ts[:50]
    pos2, last2 = Fn.hstu_cache_append(st2._struct(), ids2.to(DEV), ts2.to(DEV), bad.to(DEV), 16)
    want2 = jr.cache_append_packed(ids2, ts2, bad, 16, None, None, torch.zeros(4, dtype=torch.int32), torch.zeros(4, dtype=torch.uint8), 80)
    assert torch.equal(pos2.cpu(), want2["positions"]) and torch.equal(last2.cpu(), want2["last_row"])
    # a pool: the allocation counts each sequence's items; a rejected user, a repeated one and exhaustion of the free stack
    pool = m.new_pool(max_users=8, num_pages=5, page_size=64, max_items=192)
    users = torch.tensor([6, 2, 11, 2, 0], dtype=torch.int64)
    ids3, ts3, off3 = jr.random_packed_chunk(g, 5, 130, V, idle=4, lengths=[130, 70, 5, 9, 120], zero_frac=0.0)
    pt0, stack0 = pool.page_table.cpu(), pool.free_stack.cpu()
    pos3, last3, room3 = Fn.hstu_pool_append(pool._struct(), users.to(DEV), ids3.to(DEV), ts3.to(DEV), off3.to(DEV), 130)
    alloc = er.pool_alloc(users, jr.packed_counts(ids3, off3, 130), torch.zeros(8, dtype=torch.int32), pt0, stack0, 5, 8, 192, 64)
    assert torch.equal(room3.cpu(), alloc["room"]) and torch.equal(pool.page_table.cpu(), alloc["page_table"])
    assert int(pool.free_top) == alloc["free_top"] and int(pool.error_bits) == alloc["errors"] == er.POOL_ERR_RANGE | er.POOL_ERR_REPEAT
    want3 = jr.padded_equivalent(ids3, ts3, off3, 130, users, alloc["room"], torch.zeros(8, dtype=torch.int32),
                                 torch.zeros(8, dtype=torch.uint8), 192)
    assert torch.equal(pos3.cpu(), want3["positions"]) and torch.equal(last3.cpu(), want3["last_row"])
    assert torch.equal(pool.lengths.cpu(), want3["lengths"]) and torch.equal(pool.overflow.cpu(), want3["overflow"])
    assert bool(want3["overflow"].any())           # the free stack ran out: items were dropped in row order


# ---------------------------------------------------------------------------------------------------------------- attention vs fp64
def test_packed_chunk_attention_vs_fp64():
    """One block's packed chunk attention (the O of the workspace) against attention_rows in fp64, on rows whose query tiles cross
    64 rows, with keys split over several CTAs and histories that cross pages; the test checks those edges are reached."""
    import ctypes as C
    import genrec_b200.functional as Fn
    from genrec_b200 import _lib
    from genrec_b200._lib import check, ptr, stream_ptr
    from genrec_b200.hstu import _thresholds_on
    from tests import hstu_block_reference as hr
    m = _model(128, 4)
    layer = m.layers[0]
    H, D = 4, 128
    pool = m.new_pool(max_users=6, num_pages=60, page_size=64, max_items=1024)
    users = Users(6, seed=2)
    hist = [300, 0, 129, 64, 700, 5]
    items, stamps = users.chunk(hist, zero_frac=0.0)
    ids, ts, off = packed(items, stamps)
    m.extend_users_jagged(pool, torch.arange(6, device=DEV), ids, off, max(hist), ts)
    lens = [70, 1, 0, 65, 130, 64]                   # query tiles crossing 64 rows, an empty sequence
    items, stamps = users.chunk(lens, zero_frac=0.0)
    ids, ts, off = packed(items, stamps, idle=7)
    us = torch.tensor([4, 1, 3, 0, 2, 5], device=DEV)
    max_len = max(lens)
    cache = pool._struct()
    pos, _, _ = Fn.hstu_pool_append(cache, us, ids, ts, off, max_len)
    T = ids.numel()
    x = torch.randn(T, D, device=DEV)
    dims = Fn._dims(len(lens), max_len, D, H, layer.position_bias.num_buckets, layer.temporal_bias.num_buckets, 0.0, 0, None, 0)
    lib = _lib.load()
    nbytes = lib.grb_hstu_layer_extend_paged_workspace_bytes_jagged(C.byref(dims), C.byref(cache), T)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=DEV)
    y = torch.empty_like(x)
    pst = Fn._layer_param_struct(layer._params(), layer._bf16_weights(), True)
    uniform, b0 = layer.position_bias.uniform_of(1024, DEV)
    with torch.cuda.device(DEV):
        check(lib.grb_hstu_layer_extend_paged_jagged(C.byref(dims), C.byref(pst), C.byref(cache), 0, ptr(us), ptr(off), T, ptr(pos),
                                                     None, int(b0), ptr(_thresholds_on(DEV)), ptr(x), ptr(y), ptr(ws),
                                                     stream_ptr(DEV)))
    torch.cuda.synchronize()
    lay = hr.saved_layout(T, D)
    P, O = hr.view(ws, lay, "P"), hr.view(ws, lay, "O")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    split = er.extend_split(len(lens), max_len, H, 1024, sms)
    lengths = pool.lengths.cpu()
    K = int(lengths.max())
    offs = off.cpu().tolist()
    reached = set()
    for b, u in enumerate(us.tolist()):
        n = lens[b]
        if n == 0:
            continue
        rows = slice(offs[b], offs[b] + n)
        p = pos[rows].cpu()[None]
        kr, ok = er.cache_rows(torch.tensor([u]), lengths[u:u + 1], K, pool.page_table.cpu(), 64)
        kv = pool.kv[0].view(-1, 2 * D)[kr.to(DEV)].cpu()
        tk = pool.timestamps.view(-1)[kr.to(DEV)].cpu()
        wpos = layer.position_bias.relative_attention_bias.weight.detach().cpu()[b0:b0 + 1]
        w = er.cell_bias(p, K, wpos, None, layer.temporal_bias.temporal_attention_bias.weight.detach().cpu(), ts[rows].cpu()[None], tk,
                         _thresholds_on("cpu"), layer.temporal_bias.num_buckets)
        valid = (torch.arange(K)[None, None, :] <= p[..., None]) & ok[:, None, :]
        ref = er.attention_rows(P[rows].cpu()[None, :, 2 * D:3 * D], kv[..., :D], kv[..., D:], w, valid, er.row_depth(p, split), H)
        worst = dr.worst(O[rows].cpu(), ref["O"][0], ref["a_O"][0])
        assert worst <= dr.TOL, (b, worst)
        if n > 64:
            reached.add("query tile crossing 64 rows")
        if int(p.max()) >= split:
            reached.add("multi-split keys")
        if int(p.max()) // 64 > int(p.min()) // 64:      # the chunk's own rows straddle two pages
            reached.add("page boundary")
    assert reached == {"query tile crossing 64 rows", "multi-split keys", "page boundary"}, reached
    # idle rows have no position and an O of zero
    idle = slice(offs[-1], T)
    assert bool((pos[idle] == -1).all()) and bool((O[idle] == 0).all())


# ---------------------------------------------------------------------------------------------------------------- contract 2
@pytest.mark.parametrize("target", ["state", "pool"])
def test_packed_prefill_equals_full_forward_non_uniform(monkeypatch, target):
    """Packed prefills under the sign-fixed (non-uniform) position buckets give last_logits of the left-padded batch within the
    extend tests' oracle budget: a packed chunk has no pads ahead of a user's items."""
    m = _model(64, 2, seed=7)
    _sign_fixed(m)
    use_sign_fixed_oracle(monkeypatch)
    assert not m.layers[0].position_bias.uniform_of(200, DEV)[0]
    lens = [1, 50, 64, 0, 33, 64]
    items, stamps = Users(6, seed=3).chunk(lens, zero_frac=0.0)
    ids, ts, off = packed(items, stamps, idle=4)
    pi, pt = padded(items, stamps, 64)
    if target == "state":
        ext = m.extend_jagged(m.new_state(6, 64), ids, off, 64, ts)
    else:
        ext = m.extend_users_jagged(m.new_pool(8, 16, 64, 128), [5, 0, 2, 7, 1, 3], ids, off, 64, ts)
    _check(ext, m, pi, pt, [b for b, n in enumerate(lens) if n])


# ---------------------------------------------------------------------------------------------------------------- contract 3
def test_idle_rows_and_empty_sequences_change_nothing():
    """The same chunk with and without idle rows (junk ids and timestamps) gives the same bits; a user with an empty sequence keeps
    their cache and their previous output row."""
    m = _model(128, 4)
    users = Users(4, seed=9)
    sa, sb = m.new_state(4, 200), m.new_state(4, 200)
    items, stamps = users.chunk([20, 3, 9, 40])
    for s in (sa, sb):
        ids, ts, off = packed(items, stamps)
        m.extend_jagged(s, ids, off, 40, ts)
    before = [t.clone() for t in state_tensors(sb)]
    items, stamps = users.chunk([5, 0, 0, 2])
    ids, ts, off = packed(items, stamps)
    want = m.extend_jagged(sa, ids, off, 5, ts)
    ids, ts, off = packed(items, stamps, idle=61, seed=4)
    got = m.extend_jagged(sb, ids, off, 5, ts)
    assert torch.equal(got, want)
    for x, y in zip(state_tensors(sa), state_tensors(sb)):
        assert torch.equal(x, y)
    for b in (1, 2):
        assert torch.equal(sb.kv[:, b], before[0][:, b]) and torch.equal(sb.last_hidden[b], before[4][b])
        assert torch.equal(got[b], m._hidden_logits(before[4][b:b + 1])[0])


# ---------------------------------------------------------------------------------------------------------------- contract 4
def test_device_user_rules_match_the_padded_call():
    """Device users out of range or repeated count as empty and set errors(); items beyond max_items or without a free page are
    dropped in row order and flag their users - exactly as the padded call does it."""
    m = _model(64, 2)
    a, b = (m.new_pool(max_users=6, num_pages=6, page_size=64, max_items=256) for _ in range(2))
    users = Users(9, seed=1)
    for k, (us, lens) in enumerate([([0, 9, 1, 0, -3, 2], [100, 5, 130, 7, 2, 64]), ([2, 1, 3, 4], [200, 64, 40, 1])]):
        items, stamps = users.chunk(lens)
        u = torch.tensor(us, device=DEV)
        pi, pt = padded(items, stamps, max(lens))
        want = m.extend_users(b, u, pi, pt, num_candidates=50)
        ids, ts, off = packed(items, stamps, idle=2)
        got = m.extend_users_jagged(a, u, ids, off, max(lens), ts, num_candidates=50)
        assert_same(got, want, k)
        for x, y in zip(pool_tensors(a), pool_tensors(b)):
            assert torch.equal(x, y), k
    assert int(a.errors()) == a.ERR_USER_RANGE | a.ERR_USER_REPEAT
    assert bool(a.overflowed().any()) and int(a.pages_free()) == 0


# ---------------------------------------------------------------------------------------------------------------- selection
@pytest.mark.parametrize("mode", ["top_k", "num_candidates", "top_k_exclude", "candidates_exclude"])
def test_selection_keywords_equal_the_padded_call(mode):
    m = _model(128, 4)
    sa, sb = m.new_state(3, 100), m.new_state(3, 100)
    pa, pb = (m.new_pool(5, 12, 64, 128) for _ in range(2))
    users = Users(3, seed=6)
    kw = {"top_k": dict(top_k=20), "num_candidates": dict(num_candidates=300),
          "top_k_exclude": dict(top_k=20, exclude=torch.randint(0, V, (3, 40), device=DEV)),
          "candidates_exclude": dict(num_candidates=300, exclude=torch.randint(0, V, (3, 40), device=DEV))}[mode]
    for lens in ([30, 0, 64], [2, 5, 1]):
        items, stamps = users.chunk(lens)
        n = max(lens)
        pi, pt = padded(items, stamps, n)
        ids, ts, off = packed(items, stamps, idle=1)
        assert_same(m.extend_jagged(sa, ids, off, n, ts, **kw), m.extend(sb, pi, pt, **kw))
        assert_same(m.extend_users_jagged(pa, [4, 0, 2], ids, off, n, ts, **kw), m.extend_users(pb, [4, 0, 2], pi, pt, **kw))


# ---------------------------------------------------------------------------------------------------------------- host bounds
def test_host_bounds_for_cpu_and_device_offsets():
    m = _model(64, 2)
    st = m.new_state(3, 100)
    items, stamps = Users(3, seed=2).chunk([10, 0, 4])
    ids, ts, off = packed(items, stamps, offsets_on="cpu")
    m.extend_jagged(st, ids, off, 40, ts)
    assert st.items_bound == 10                      # the longest CPU length
    m.extend_jagged(st, ids, off.to(DEV), 40, ts)
    assert st.items_bound == 50                      # max_len: device offsets are not read on the host
    with pytest.raises(ValueError, match="capacity"):
        m.extend_jagged(st, ids, off.to(DEV), 51, ts)
    pool = m.new_pool(6, 8, 64, 128)
    m.extend_users_jagged(pool, [4, 0, 2], ids, off, 40, ts)
    assert pool.items_bound.tolist() == [0, 0, 4, 0, 10, 0] and pool.pages_bound == 2
    m.extend_users_jagged(pool, [4, 0, 2], ids, off.to(DEV), 40, ts)
    assert pool.items_bound.tolist() == [40, 0, 44, 0, 50, 0] and pool.pages_bound == 3
    m.extend_users_jagged(pool, torch.tensor([4, 0, 2], device=DEV), ids, off.to(DEV), 40, ts)
    assert pool.items_bound.tolist() == [40, 0, 44, 0, 50, 0]       # device users: no host bookkeeping
    with pytest.raises(ValueError, match="max_items"):
        m.extend_users_jagged(pool, [4, 0, 2], ids, off.to(DEV), 90, ts)


# ---------------------------------------------------------------------------------------------------------------- CUDA graphs
def test_cuda_graph_replay_with_rewritten_offsets_ids_and_users():
    """A packed extend_users_jagged with fixed (B, T, max_len) and device users / offsets, captured after one eager call, replays
    with rewritten offsets, ids, timestamps and users exactly as eager calls on a twin pool."""
    m = _model(128, 4)
    eager, graphed = (m.new_pool(max_users=8, num_pages=40, page_size=64, max_items=256) for _ in range(2))
    B, T, max_len = 4, 48, 12
    users = Users(8, seed=4)
    gen = torch.Generator().manual_seed(7)

    def draw():
        lens = torch.randint(0, max_len + 1, (B,), generator=gen).tolist()
        us = torch.randperm(8, generator=gen)[:B]
        all_lens = [0] * 8
        for u, n in zip(us.tolist(), lens):
            all_lens[u] = n
        items, stamps = users.chunk(all_lens)
        items, stamps = [items[u] for u in us.tolist()], [stamps[u] for u in us.tolist()]
        ids, ts, off = packed(items, stamps, idle=T - sum(lens), seed=int(us[0]))
        return us.to(DEV), ids, ts, off

    s_users, s_ids, s_ts, s_off = draw()
    m.extend_users_jagged(eager, s_users, s_ids, s_off, max_len, s_ts, top_k=10)
    m.extend_users_jagged(graphed, s_users, s_ids, s_off, max_len, s_ts, top_k=10)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = m.extend_users_jagged(graphed, s_users, s_ids, s_off, max_len, s_ts, top_k=10)
    for step in range(5):
        us, ids, ts, off = draw()
        ref = m.extend_users_jagged(eager, us, ids, off, max_len, ts, top_k=10)
        s_users.copy_(us)
        s_ids.copy_(ids)
        s_ts.copy_(ts)
        s_off.copy_(off)
        g.replay()
        torch.cuda.synchronize()
        assert_same(tuple(out), tuple(ref), step)
        for a, b in zip(pool_tensors(graphed), pool_tensors(eager)):
            assert torch.equal(a, b), step


# ---------------------------------------------------------------------------------------------------------------- recommend / retrieve
def _hstu_rec_model():
    from genrec_b200.hstu import HSTU
    torch.manual_seed(0)
    m = HSTU(V, 200, 64, 2, 2, dropout=0.0).to(DEV).eval()
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "attention_bias" in n:
                p.normal_(0, 0.3)
    return m


def _check_selection(sel, logits, k):
    """TopItems whose scores are the logits of their items, bit for bit, and are the row's k best (item 0 left out)."""
    assert torch.equal(sel.scores, logits.gather(1, sel.items))
    masked = logits.clone()
    masked[:, 0] = float("-inf")
    assert torch.equal(sel.scores, masked.topk(k, dim=1).values)


@pytest.mark.parametrize("which", ["recommend", "retrieve"])
def test_hstu_recommend_and_retrieve_jagged(which):
    import genrec_b200.functional as Fn
    m = _hstu_rec_model()
    lens = [0, 1, 63, 64, 65, 17]
    items, stamps = Users(6, seed=8).chunk(lens, zero_frac=0.0)
    ids, ts, off = packed(items, stamps, idle=5)
    k = 10 if which == "recommend" else 300
    sel = (m.recommend_jagged(ids, off, 65, ts, top_k=k) if which == "recommend" else m.retrieve_jagged(ids, off, 65, ts, num_candidates=k))
    hidden = Fn.last_rows_jagged(m.encode_jagged(ids, off, 65, ts), off)
    assert torch.equal(hidden[0], torch.zeros_like(hidden[0]))           # the empty sequence: the head of a zero vector
    _check_selection(sel, m._hidden_logits(hidden), k)
    pi, pt = padded(items, stamps, 65)
    want = m.recommend(pi, pt, top_k=k) if which == "recommend" else m.retrieve(pi, pt, num_candidates=k)
    real = [b for b, n in enumerate(lens) if n]
    assert relerr(sel.scores[real], want.scores[real]) <= PACKED_VS_PADDED_TOL


@pytest.mark.parametrize("which", ["recommend", "retrieve"])
def test_sasrec_recommend_and_retrieve_jagged(which):
    """SASRec's packed batch keeps its batch-wide position rule: the left-padded batch it equals is padded to the longest
    sequence, P, whatever max_len is."""
    import genrec_b200.functional as Fn
    from genrec_b200.sasrec import SASRec
    torch.manual_seed(0)
    m = SASRec(V, 50, 64, 2, 2, 256, dropout=0.0).to(DEV).eval()
    lens = [0, 1, 9, 33, 17]
    items, _ = Users(5, seed=2).chunk(lens, zero_frac=0.0)
    ids, _, off = packed(items, [torch.zeros(n, dtype=torch.int64) for n in lens], idle=3)
    k = 10 if which == "recommend" else 400
    sel = m.recommend_jagged(ids, off, 50, top_k=k) if which == "recommend" else m.retrieve_jagged(ids, off, 50, num_candidates=k)
    hidden = Fn.last_rows_jagged(m.encode_jagged(ids, off, 50), off)
    logits = Fn.head_logits(hidden[:, None, :], m.final_norm.weight, m.final_norm.bias, m.item_embedding.weight,
                            Fn.cast_bf16(m.item_embedding.weight), m.final_norm.eps)[:, 0, :]
    _check_selection(sel, logits, k)
    P = max(lens)
    pi, _ = padded(items, [torch.zeros(n, dtype=torch.int64) for n in lens], P)
    want = m.recommend(pi, top_k=k) if which == "recommend" else m.retrieve(pi, num_candidates=k)
    real = [b for b, n in enumerate(lens) if n]
    assert relerr(sel.scores[real], want.scores[real]) <= PACKED_VS_PADDED_TOL
