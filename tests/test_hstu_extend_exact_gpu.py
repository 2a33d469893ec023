"""One HSTU layer's cached extend through the C ABI, on caches and a workspace this module owns, against the references of
tests/extend_reference.py, at the shapes serving runs: key splits of many 64-key tiles (up to a whole 2,048-item history in one
CTA), splits that cross pages, start in the middle of a page or are cut short by the capacity, 256 partials of one tile each, a
16,384-item prefill in one call, and calls of more than 1,024 users, whose page bookkeeping runs in several 1,024-row chunks.

Every call is checked on the kernel's own inputs: the bookkeeping of grb_hstu_pool_append / grb_hstu_cache_append against the
integer restatement (bit for bit), the K | V rows the extend scatters against the workspace's P (bit for bit, every other cache row
unchanged), and O of every queried row against the fp64 attention of the workspace's Q over the K | V and timestamps gathered back
through the page table (tolerance dense_reference.TOL on the derived allowance).  The workspace starts as 0xFF bytes (NaN), so an
unwritten partial or O row shows.  `pytest -s` prints the worst error / allowance of each checked quantity."""
import ctypes as C

import pytest
import torch

from tests import extend_reference as er
from tests import hstu_block_reference as hr
from tests.exact_check import Ledger, _sms
from tests.hstu_cases import _params, batch, pos_fixed

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
NPOS, MAXD, NTIME = 32, 100, 64
INT_MAX = (1 << 31) - 1
LEDGER = Ledger("worst error / allowance per quantity (tolerance 1):")
_error_table = LEDGER.fixture()
_check = LEDGER.check


# ------------------------------------------------------------------------------------------------ caches the test owns
def _timestamps(total, wide, g):
    """increasing timestamps of one user's `total` items: day-scale gaps with repeats, or (wide) gaps spanning ~2^62 in all"""
    if wide:
        return 1_300_000_000 + torch.arange(total, dtype=torch.int64) * ((1 << 62) // max(total, 1))
    gaps = torch.randint(0, 3 * 86400, (total,), generator=g)
    gaps[::4] = 0
    return 1_300_000_000 + torch.cumsum(gaps, 0)


class Cache:
    """One layer's K | V cache: a pool (page table, scrambled free stack) or the dense [B, cap] state, with every row of kv and
    timestamps random so that a read of a wrong row shows."""

    def __init__(self, D, hist, ts, g, cap, page_size=None, max_users=None, spare_pages=4):
        """hist: {user: K | V rows [len, 2D] bf16}, ts: {user: timestamps [len]}; page_size None: the dense cache of users 0 ..
        len(hist) - 1."""
        self.D, self.cap, self.ps = D, cap, page_size
        self.dense = page_size is None
        if self.dense:
            self.B = len(hist)
            nrows = self.B * cap
            self.lengths = torch.tensor([len(hist[u]) for u in range(self.B)], dtype=torch.int32)
        else:
            self.max_users = max_users
            self.pt_ld = -(-cap // page_size)
            held = {u: -(-len(hist[u]) // page_size) for u in hist}
            self.num_pages = sum(held.values()) + spare_pages
            nrows = self.num_pages * page_size
            perm = torch.randperm(self.num_pages, generator=g).to(torch.int32)
            self.page_table = torch.zeros(max_users, self.pt_ld, dtype=torch.int32)
            k = 0
            for u in sorted(hist, key=lambda _: int(torch.randint(0, 1 << 30, (1,), generator=g))):
                self.page_table[u, :held[u]] = perm[k:k + held[u]]
                k += held[u]
            self.free_stack = torch.full((self.num_pages,), -5, dtype=torch.int32)
            self.free_stack[:self.num_pages - k] = perm[k:]
            self.free_top = torch.tensor([self.num_pages - k], dtype=torch.int32)
            self.errors = torch.zeros(1, dtype=torch.int32)
            self.row_of = torch.full((max_users,), INT_MAX, dtype=torch.int32)
            self.lengths = torch.zeros(max_users, dtype=torch.int32)
            for u in hist:
                self.lengths[u] = len(hist[u])
        self.overflow = torch.zeros(len(self.lengths), dtype=torch.uint8)
        self.kv = torch.nn.functional.silu(0.7 * torch.randn(nrows, 2 * D, generator=g)).bfloat16()
        self.ts = torch.randint(0, 1 << 40, (nrows,), generator=g)
        for u in hist:
            r = self.rows(torch.tensor([u]), torch.tensor([len(hist[u])], dtype=torch.int32), len(hist[u]))[0][0]
            self.kv[r] = hist[u]
            self.ts[r] = ts[u]
        for name in self.tensors():
            setattr(self, name, getattr(self, name).to(DEV))

    def tensors(self):
        base = ["kv", "ts", "lengths", "overflow"]
        return base if self.dense else base + ["page_table", "free_stack", "free_top", "errors", "row_of"]

    def snapshot(self):
        return {n: getattr(self, n).clone() for n in self.tensors()}

    def struct(self):
        from genrec_b200._lib import HstuCache, HstuPool, ptr
        if self.dense:
            return HstuCache(self.B, self.cap, 1, ptr(self.kv), ptr(self.ts), ptr(self.lengths), ptr(self.overflow))
        return HstuPool(self.max_users, 1, self.ps, self.num_pages, self.cap, ptr(self.kv), ptr(self.ts), ptr(self.page_table),
                        ptr(self.lengths), ptr(self.overflow), ptr(self.free_stack), ptr(self.free_top), ptr(self.errors),
                        ptr(self.row_of))

    def rows(self, users, lengths, K, page_table=None):
        """[B, K] cache row of item j of each user (0 beyond its length) and the mask j < length"""
        if self.dense:
            return er.cache_rows(users, lengths, K, cap=self.cap)
        pt = self.page_table if page_table is None else page_table
        return er.cache_rows(users.to(pt.device), lengths.to(pt.device), K, pt, self.ps)

    def gather(self, users, K):
        """K | V [B, K, 2D] and timestamps [B, K] of items 0 .. K-1 of each user, read through the page table"""
        r, ok = self.rows(users, self.lengths[users.to(DEV)], K)
        return self.kv[r], self.ts[r], ok


# ------------------------------------------------------------------------------------------------ one call: append + extend
def append(cache, users, ids, ts):
    """grb_hstu_pool_append / grb_hstu_cache_append, checked against the restatement bit for bit.  -> positions, last_row"""
    from genrec_b200 import _lib
    from genrec_b200._lib import check, ptr, stream_ptr
    lib = _lib.load()
    B, n = ids.shape
    before = cache.snapshot()
    lens0, ov0 = before["lengths"].cpu(), before["overflow"].cpu()
    room = None
    if not cache.dense:
        ref = er.pool_alloc(users, (ids != 0).sum(1), lens0, before["page_table"].cpu(), before["free_stack"].cpu(),
                            int(before["free_top"]), cache.max_users, cache.cap, cache.ps)
        room = ref["room"]
    app = er.cache_append(ids, ts, None if cache.dense else users, room, lens0, ov0, cache.cap)
    positions = torch.full((B, n), -7, dtype=torch.int32, device=DEV)
    last_row = torch.full((B,), -7, dtype=torch.int32, device=DEV)
    idc, tsc = ids.to(DEV), ts.to(DEV)
    st = cache.struct()
    if cache.dense:
        check(lib.grb_hstu_cache_append(C.byref(st), ptr(idc), ptr(tsc), n, ptr(positions), ptr(last_row), stream_ptr(DEV)))
    else:
        room_d = torch.full((B,), -7, dtype=torch.int32, device=DEV)
        uc = users.to(DEV)
        check(lib.grb_hstu_pool_append(C.byref(st), ptr(uc), B, ptr(idc), ptr(tsc), n, ptr(positions), ptr(last_row), ptr(room_d),
                                       stream_ptr(DEV)))
    torch.cuda.synchronize()
    assert torch.equal(positions.cpu(), app["positions"]), "positions"
    assert torch.equal(last_row.cpu(), app["last_row"]), "last_row"
    assert torch.equal(cache.lengths.cpu(), app["lengths"]), "lengths"
    assert torch.equal(cache.overflow.cpu(), app["overflow"]), "overflow"
    if not cache.dense:
        assert torch.equal(room_d.cpu(), ref["room"]), "room"
        assert torch.equal(cache.page_table.cpu(), ref["page_table"]), "page_table"
        assert int(cache.free_top) == ref["free_top"], "free_top"
        assert int(cache.errors) == ref["errors"], "errors"
        assert torch.equal(cache.free_stack, before["free_stack"]), "the allocation rewrote the free stack"
        assert bool((cache.row_of == INT_MAX).all()), "row_of not restored"
    want_ts = before["ts"].clone()
    if app["writes"]:
        u, q, t = (torch.tensor(c) for c in zip(*app["writes"]))
        r = _row_of(cache, u, q)
        want_ts[r] = t.to(DEV)
    assert torch.equal(cache.ts, want_ts), "timestamps: a wrong row written or a row missed"
    assert torch.equal(cache.kv, before["kv"]), "the append wrote K | V"
    return positions


def _row_of(cache, u, q):
    if cache.dense:
        return (u * cache.cap + q).to(DEV)
    pt = cache.page_table.long()
    u, q = u.to(DEV), q.to(DEV)
    return pt[u, q // cache.ps] * cache.ps + q % cache.ps


def extend(cache, users, positions, x, prm, H, uniform, timed, case, sample=None):
    """grb_hstu_layer_extend(_paged) of one layer; checks the scatter, the untouched rows and O.  -> O, y, the workspace's P"""
    from genrec_b200 import _lib
    from genrec_b200._lib import HstuDims, HstuLayerParams, check, ptr, stream_ptr
    from genrec_b200.hstu import _thresholds_on
    lib = _lib.load()
    B, n = positions.shape
    D, cap = cache.D, cache.cap
    T = B * n
    ntime = NTIME if timed else 0
    dims = HstuDims(B, n, D, H, NPOS, ntime, 0.0, 0, None, 0)
    names = ("proj_w", "proj_b", "pos_table", "time_table", "ln1_g", "ln1_b", "ffn1_w", "ffn1_b", "ffn2_w", "ffn2_b", "ln2_g", "ln2_b")
    pst = HstuLayerParams(*[ptr(prm[k]) if (k != "time_table" or timed) else None for k in names])
    pb0 = 3
    pos_bucket = None if uniform else pos_fixed(torch.arange(cap), NPOS, MAXD).to(torch.uint8).to(DEV)
    thr = _thresholds_on(DEV)
    st = cache.struct()
    if cache.dense:
        nbytes = lib.grb_hstu_layer_extend_workspace_bytes(C.byref(dims), cap)
    else:
        nbytes = lib.grb_hstu_layer_extend_paged_workspace_bytes(C.byref(dims), C.byref(st))
    split = er.extend_split(B, n, H, cap, _sms())
    assert nbytes == er.extend_workspace_bytes(B, n, D, H, cap, _sms()), (nbytes, case)
    ws = torch.full((nbytes,), 0xFF, dtype=torch.uint8, device=DEV)
    y = torch.full((T, D), float("nan"), device=DEV)
    before = cache.snapshot()
    args = (ptr(pos_bucket), pb0, ptr(thr), ptr(x), ptr(y), ptr(ws), stream_ptr(DEV))
    if cache.dense:
        check(lib.grb_hstu_layer_extend(C.byref(dims), C.byref(pst), C.byref(st), 0, ptr(positions), *args))
    else:
        uc = users.to(DEV)
        check(lib.grb_hstu_layer_extend_paged(C.byref(dims), C.byref(pst), C.byref(st), 0, ptr(uc), ptr(positions), *args))
    torch.cuda.synchronize()
    sl = hr.saved_layout(T, D)
    P, O = hr.view(ws, sl, "P"), hr.view(ws, sl, "O")
    assert bool(torch.isfinite(y).all()), case
    # scatter: the chunk's K | V rows land where the positions say, nothing else moves
    pos = positions.view(-1).long()
    live = pos >= 0
    brow = torch.arange(B, device=DEV).repeat_interleave(n)[live]
    u_of = brow if cache.dense else users.to(DEV)[brow]
    want_kv = before["kv"].clone()
    want_kv[_row_of(cache, u_of, pos[live])] = torch.cat([P[live, 3 * D:], P[live, D:2 * D]], 1)
    assert torch.equal(cache.kv, want_kv), f"{case}: scattered K | V rows differ from P, or another cache row changed"
    for name in cache.tensors():
        if name != "kv":
            assert torch.equal(getattr(cache, name), before[name]), f"{case}: the extend changed {name}"
    # O: rows without a position are exactly 0; the queried rows against the fp64 attention on the kernel's own inputs
    pos2 = positions.long()
    assert not bool(O.view(B, n, D)[pos2 < 0].any()), f"{case}: O of a row without a position is not 0"
    # the combine: O = bf16 of the fp32 sum of the row's split partials, added in split order, bit for bit
    nsplit = -(-cap // split)
    part = ws[sl["bytes"]:sl["bytes"] + nsplit * T * D * 4].view(torch.float32).view(nsplit, T, D)
    acc = torch.zeros(T, D, device=DEV)
    for s in range(nsplit):
        acc = torch.where((live & (pos // split >= s))[:, None], acc + part[s], acc)
    assert torch.equal(O, acc.bfloat16()), f"{case}: O is not the split-ordered sum of the partials"
    rows = torch.arange(n, device=DEV) if sample is None else sample.to(DEV)
    pr = pos2[:, rows]
    K = int(pr.max()) + 1
    kvg, tsg, _ = cache.gather(users if users is not None else torch.arange(B), K)
    tq = torch.gather(tsg, 1, pr.clamp_min(0))
    wpos = prm["pos_table"][pb0:pb0 + 1] if uniform else prm["pos_table"]
    w = er.cell_bias(pr, K, wpos, pos_bucket, prm["time_table"][:NTIME] if timed else None, tq, tsg, thr, NTIME)
    valid = torch.arange(K, device=DEV)[None, None, :] <= pr[:, :, None]
    Q = P.view(B, n, 4 * D)[:, rows, 2 * D:3 * D]
    at = er.attention_rows(Q, kvg[..., :D], kvg[..., D:], w, valid, er.row_depth(pr, split), H)
    live_r = pr >= 0
    _check(case, [("extend O", O.view(B, n, D)[:, rows][live_r], at["O"][live_r], at["a_O"][live_r])])
    return O.clone(), y, P.clone()


# ------------------------------------------------------------------------------------------------ the case table
# (name, B, D, H, n, capacity, page_size (None: dense), uniform position buckets, time term)
CASES = [
    ("one-cta", 132, 128, 4, 1, 2048, 64, True, True),          # split 2,048: the whole history in one CTA, 32 tiles and pages
    ("cfg3-pool", 32, 256, 8, 1, 2048, 64, False, True),        # split 704, 3 splits, the last cut short at 2,048
    ("cfg2-pool", 128, 128, 4, 1, 200, 64, True, False),        # split 128, 2 splits
    ("mid-page", 64, 256, 4, 1, 1000, 256, False, False),       # split 384: splits 1 and 2 start in the middle of a page
    ("two-qtiles", 40, 128, 4, 65, 700, 192, False, True),      # 2 query tiles, split 384 over two 192-item pages
    ("partials", 1, 128, 2, 64, 16384, None, True, True),       # split 64: 256 partials of one tile each
    ("prefill", 1, 128, 2, 16384, 16384, None, False, True),    # split 8,192: 128 tiles per CTA
    ("over-1024", 1100, 64, 2, 1, 192, 64, True, False),        # B > 1,024: the bookkeeping's chunk loop
]


def _not_64(v, lo, hi, g):
    while v % 64 == 0:
        v = int(torch.randint(lo, hi + 1, (1,), generator=g))
    return v


def _case_state(B, D, n, cap, ps, g):
    """history lengths, K | V rows and timestamps of the call's users (rows 1 / 2 / 3 of a one-item call: a history that reaches
    the last key, a full one whose item overflows, an empty one), a chunk with all-pad rows and pads, and the users: a random
    subset of max_users = B + 5 (the other five hold pages too)."""
    max_users = B + 5
    users = torch.randperm(max_users, generator=g)[:B] if ps else torch.arange(B)
    lens, hi = {}, cap - n
    for b in range(B):
        lens[b] = _not_64(int(torch.randint(1, hi + 1, (1,), generator=g)), 1, hi, g) if hi >= 1 else 0
    if n == 1 and B > 3:
        lens[1], lens[2], lens[3] = cap - 1, cap, 0
    if n == 64:
        lens[0] = cap - n - 37
    if n == cap:
        lens[0] = 0
    ids = torch.randint(1, 500, (B, n), generator=g)
    for b in range(B):
        if b % 7 == 5 and B > 1:
            ids[b] = 0                                          # all padding
        elif n > 1:
            ids[b, :b % 5] = 0                                  # left pads
            ids[b, torch.randint(0, n, (max(1, n // 300),), generator=g)] = 0       # pads inside the chunk
    hist, hts, cts = {}, {}, torch.zeros(B, n, dtype=torch.int64)
    for b in range(B):
        full = _timestamps(lens[b] + n, wide=b % 5 == 3, g=g)
        u = int(users[b])
        hist[u] = torch.nn.functional.silu(0.7 * torch.randn(lens[b], 2 * D, generator=g)).bfloat16()
        hts[u] = full[:lens[b]]
        cts[b] = torch.where(ids[b] != 0, full[lens[b]:], torch.zeros(n, dtype=torch.int64))
    if ps:
        for u in range(max_users):
            if u not in hist:
                L = _not_64(int(torch.randint(1, cap + 1, (1,), generator=g)), 1, cap, g)
                hist[u] = torch.nn.functional.silu(0.7 * torch.randn(L, 2 * D, generator=g)).bfloat16()
                hts[u] = _timestamps(L, False, g)
    return users, ids, cts, hist, hts, max_users


def _prefill_sample(positions, split, g):
    """chunk rows to check of the one-call prefill: those at a split boundary (positions k split - 1 and k split), the last 64 rows
    and 200 random rows"""
    p = positions[0].cpu().long()
    edge = torch.zeros_like(p, dtype=torch.bool)
    for k in range(1, int(p.max()) // split + 1):
        edge |= (p == k * split - 1) | (p == k * split)
    edge[-64:] = True
    edge[torch.randint(0, p.numel(), (200,), generator=g)] = True
    return torch.nonzero(edge).view(-1)


def run_case(name, B, D, H, n, cap, ps, uniform, timed, seed):
    g = torch.Generator().manual_seed(seed)
    users, ids, cts, hist, hts, max_users = _case_state(B, D, n, cap, ps, g)
    spare = sum(-(-(len(hist[int(u)]) + n) // ps) for u in users) if ps else 0
    cache = Cache(D, hist, hts, g, cap, ps, max_users, spare_pages=spare)
    prm = _params(D, H, NPOS, NTIME, seed + 1)
    positions = append(cache, users, ids, cts)
    x = torch.randn(B * n, D, generator=g).to(DEV)
    sample = _prefill_sample(positions, er.extend_split(B, n, H, cap, _sms()), g) if n > 1024 else None
    return cache, users, positions, extend(cache, users if ps else None, positions, x, prm, H, uniform, timed,
                                           f"{name} B{B} D{D} dh{D // H} n{n} cap{cap} ps{ps}", sample)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_extend_vs_fp64(case):
    run_case(*case, seed=sum(case[1:6]))


def test_edges_are_reached():
    sms = _sms()
    reg = []
    for name, B, D, H, n, cap, ps, uni, timed in CASES:
        split, ns = er.extend_split(B, n, H, cap, sms), er.extend_nsplit(B, n, H, cap, sms)
        reg.append(dict(split=split, ns=ns, tiles=split // 64, pages=split // ps if ps else 0, single=ns == 1,
                        short=ns * split > cap, mid=bool(ps) and split % ps != 0 and ns > 1, dh=D // H, cap=cap, B=B,
                        variant=(uni, timed)))
    assert any(r["split"] == 64 and r["ns"] >= 100 for r in reg)
    assert any(r["tiles"] >= 3 and r["pages"] >= 3 for r in reg)
    assert any(r["single"] for r in reg) and any(r["short"] for r in reg) and any(r["mid"] for r in reg)
    assert {32, 64} <= {r["dh"] for r in reg}
    assert any(r["cap"] == 16384 for r in reg) and any(r["B"] > 1024 for r in reg)
    assert {r["variant"] for r in reg} == {(True, True), (True, False), (False, True), (False, False)}
    from genrec_b200 import _lib
    from genrec_b200._lib import HstuDims
    lib = _lib.load()
    for name, B, D, H, n, cap, *_ in CASES:
        d = HstuDims(B, n, D, H, NPOS, NTIME, 0.0, 0, None, 0)
        assert lib.grb_hstu_layer_extend_workspace_bytes(C.byref(d), cap) == er.extend_workspace_bytes(B, n, D, H, cap, sms), name


def test_time_bucket_matches_the_bias_index_kernel():
    """er.time_bucket / er.cell_bias against the dense hstu_bias_index kernel, bit for bit, on one history whose timestamps span
    more than 2^62 in a row"""
    import genrec_b200.functional as Fn
    from genrec_b200.hstu import _thresholds_on
    L, H, ntime = 300, 2, 20
    ids, ts, pad = batch(L, 11)
    thr = _thresholds_on(DEV)
    pb = pos_fixed(torch.arange(L), NPOS, MAXD).to(torch.uint8)
    meta = Fn.SeqMeta(pad.to(torch.uint8).to(DEV), ts.to(DEV), pb.to(DEV), thr, ntime, NPOS, (False, 0))
    g = torch.Generator().manual_seed(2)
    wpos, wtime = (0.3 * torch.randn(NPOS, H, generator=g)).to(DEV), (0.5 * torch.randn(ntime, H, generator=g)).to(DEV)
    want, masked, _, tb = hr.cell_bias(meta.bias_index, wpos, wtime, NPOS, H)
    tsd = ts.to(DEV)
    keep = ~masked[:, 0]
    got_tb = er.time_bucket(tsd[:, :, None] - tsd[:, None, :], thr, ntime)
    assert torch.equal(got_tb[keep], tb[keep])
    assert int(tb[keep].max()) == ntime - 1
    i = torch.arange(L, device=DEV)
    got = er.cell_bias(i[None].expand(4, L), L, wpos, pb.to(DEV), wtime, tsd, tsd, thr, ntime)
    keep4 = keep[:, None].expand_as(want)
    assert torch.equal(got[keep4], want[keep4])


# ------------------------------------------------------------------------------------------------ pool bookkeeping at B > 1,024
def test_pool_bookkeeping_over_1024_rows():
    """A 2,500-row call in permuted user order (one user repeated across the first chunk boundary, rows 7 and 1,030; one out of
    range; all-pad rows) on a stack that runs out inside the second 1,024-row chunk; then a release of 2,100 users (one repeated);
    then an extend of 1,100 users, most on the pages the release gave back, checked against fp64."""
    from genrec_b200 import _lib
    from genrec_b200._lib import check, ptr, stream_ptr
    g = torch.Generator().manual_seed(41)
    D, H, ps, cap, max_users, n = 64, 2, 64, 192, 2600, 40
    hist, hts = {}, {}
    for u in range(0, max_users, 3):                            # a third of the users hold 1 .. 150 items
        L = _not_64(int(torch.randint(1, 151, (1,), generator=g)), 1, 150, g)
        hist[u] = torch.nn.functional.silu(0.7 * torch.randn(L, 2 * D, generator=g)).bfloat16()
        hts[u] = _timestamps(L, False, g)
    B = 2500
    users = torch.randperm(max_users, generator=g)[:B]
    users[1030] = users[7]
    users[500] = max_users + 3
    ids = torch.randint(1, 500, (B, n), generator=g)
    for b in range(B):
        ids[b, :int(torch.randint(0, n, (1,), generator=g))] = 0
        if b % 11 == 4:
            ids[b] = 0
    ts = 2_000_000_000 + torch.arange(B)[:, None] * 1000 + torch.cumsum(torch.randint(0, 50, (B, n), generator=g), 1)
    # free pages: what rows 0 .. 1,499 ask for, plus one
    lens = torch.zeros(max_users, dtype=torch.int32)
    for u in hist:
        lens[u] = len(hist[u])
    big = 4 * B
    asked = er.pool_alloc(users[:1500], (ids[:1500] != 0).sum(1), lens, torch.zeros(max_users, 3, dtype=torch.int32),
                          torch.arange(big, dtype=torch.int32), big, max_users, cap, ps)
    cache = Cache(D, hist, hts, g, cap, ps, max_users, spare_pages=big - asked["free_top"] + 1)
    append(cache, users, ids, ts)
    assert int(cache.errors) == er.POOL_ERR_RANGE | er.POOL_ERR_REPEAT and int(cache.free_top) == 0
    want = torch.minimum(lens[users.clamp(0, max_users - 1)] + (ids != 0).sum(1), torch.tensor(cap))
    got = cache.lengths.cpu()[users.clamp(0, max_users - 1)]
    short = [b for b in range(B) if b not in (500, 1030) and int(got[b]) < int(want[b])]
    assert short and 1024 <= short[0] < 2048, short[:3]        # the stack runs out inside the second chunk

    # release 2,100 users, one of them twice
    rel = torch.randperm(max_users, generator=g)[:2100]
    rel[1500] = rel[3]
    cache.errors.zero_()
    top0 = int(cache.free_top)
    last_hidden = torch.randn(max_users, D, generator=g).to(DEV)
    lh0 = last_hidden.clone()
    ref = er.pool_release(rel, cache.lengths.cpu(), cache.overflow.cpu(), cache.page_table.cpu(), cache.free_stack.cpu(),
                          int(cache.free_top), max_users, cache.num_pages, ps)
    st = cache.struct()
    rd = rel.to(DEV)
    check(_lib.load().grb_hstu_pool_release(C.byref(st), ptr(rd), rel.numel(), ptr(last_hidden), D, stream_ptr(DEV)))
    torch.cuda.synchronize()
    assert torch.equal(cache.free_stack.cpu(), ref["free_stack"]) and int(cache.free_top) == ref["free_top"]
    assert torch.equal(cache.lengths.cpu(), ref["lengths"]) and torch.equal(cache.overflow.cpu(), ref["overflow"])
    assert int(cache.errors) == er.POOL_ERR_REPEAT and bool((cache.row_of == INT_MAX).all())
    gone = torch.zeros(max_users, dtype=torch.bool)
    gone[rel] = True
    assert not bool(last_hidden[gone.to(DEV)].any()) and torch.equal(last_hidden[~gone.to(DEV)], lh0[~gone.to(DEV)])

    # extend 700 released users (now on reused pages) and 400 that kept their histories
    keep = torch.nonzero(~gone).view(-1)
    call = torch.cat([rel[:700], keep[torch.randperm(keep.numel(), generator=g)[:400]]])
    call = call[torch.randperm(call.numel(), generator=g)]
    ids2 = torch.randint(1, 500, (call.numel(), 1), generator=g)
    ids2[::9] = 0
    ts2 = 3_000_000_000 + torch.arange(call.numel())[:, None]
    reused = set(ref["free_stack"][top0:ref["free_top"]].tolist())           # the pages the release pushed
    cache.errors.zero_()
    positions = append(cache, call, ids2, ts2)
    assert int(cache.errors) == 0
    new_pages = {int(cache.page_table[int(u), 0]) for u in rel[:700] if int(cache.lengths[int(u)]) > 0}
    assert new_pages and new_pages <= reused
    prm = _params(D, H, NPOS, NTIME, 43)
    x = torch.randn(call.numel(), D, generator=g).to(DEV)
    extend(cache, call, positions, x, prm, H, False, True, "bookkeeping B1100 after release")


# ------------------------------------------------------------------------------------------------ page-size invariance
def test_page_size_invariance():
    """The split depends on the capacity and the shapes only, so the same history and call give bit-identical O, y and gathered
    K | V on the dense state of capacity max_items and on pools of 64-, 128- and 256-item pages and of one page per user."""
    B, D, H, n, cap = 48, 128, 4, 3, 1000
    g = torch.Generator().manual_seed(77)
    lens = [_not_64(int(torch.randint(1, cap - n + 1, (1,), generator=g)), 1, cap - n, g) for _ in range(B)]
    lens[0] = cap - n
    rows_kv = [torch.nn.functional.silu(0.7 * torch.randn(L, 2 * D, generator=g)).bfloat16() for L in lens]
    full_ts = [_timestamps(L + n, b % 5 == 3, g) for b, L in enumerate(lens)]
    ids = torch.randint(1, 500, (B, n), generator=g)
    ids[5] = 0
    ids[7, 0] = 0
    ts = torch.stack([t[L:] for t, L in zip(full_ts, lens)]) * (ids != 0)
    prm = _params(D, H, NPOS, NTIME, 78)
    x = torch.randn(B * n, D, generator=g).to(DEV)
    pool_users = torch.randperm(B + 5, generator=g)[:B]
    out = []
    for ps in (None, 64, 128, 256, 1024):
        users = torch.arange(B) if ps is None else pool_users
        hist = {int(u): rows_kv[b] for b, u in enumerate(users)}
        hts = {int(u): full_ts[b][:lens[b]] for b, u in enumerate(users)}
        if ps:
            for u in range(B + 5):
                if u not in hist:
                    hist[u] = torch.zeros(100 + u, 2 * D).bfloat16()
                    hts[u] = _timestamps(100 + u, False, g)
        cache = Cache(D, hist, hts, torch.Generator().manual_seed(ps or 1), cap, ps, B + 5, spare_pages=B * 2)
        positions = append(cache, users, ids, ts)
        O, y, _ = extend(cache, users if ps else None, positions, x, prm, H, False, True, f"invariance ps{ps}")
        kv, t, ok = cache.gather(users, cap)
        out.append((positions, O, y, kv[ok], t[ok]))
    for ps, r in zip((64, 128, 256, 1024), out[1:]):
        for name, a, b in zip(("positions", "O", "y", "K | V", "timestamps"), r, out[0]):
            assert torch.equal(a, b), f"page_size {ps}: {name} differs from the dense state"


def test_model_extend_users_equals_extend_at_132_users():
    """HSTU.extend_users on a pool of 128-item pages (free stack scrambled by other users) against HSTU.extend on the dense state,
    at B = 132: logits bit for bit"""
    from tests.hstu_cases import _absolute_ts, _chunks, _fill, _serve_model
    m = _serve_model(128, 4, use_time=True, seed=2)
    B, cap = 132, 1000
    st = m.new_state(B, cap)
    pool = m.new_pool(max_users=150, num_pages=500, page_size=128, max_items=cap)
    _fill(m, pool, list(range(132, 150)), 200, seed=3)
    pool.release(list(range(132, 150, 2)))
    users = torch.randperm(132, generator=torch.Generator().manual_seed(4))
    for k, (ids, ts) in enumerate(_absolute_ts(_chunks(B, [300, 1, 70, 1], seed=6))):
        ref = m.extend(st, ids.cuda(), ts.cuda())
        got = m.extend_users(pool, users, ids.cuda(), ts.cuda())
        assert torch.equal(got, ref), (k, (got - ref).abs().max())
    assert not pool.overflowed().any() and int(pool.errors()) == 0
