"""fp64 and integer references of the cached extend path (csrc/attn_hstu_extend.cuh and its host plumbing in csrc/api.cu): the
chunk attention of hstu_attn_extend_kernel + hstu_extend_combine_kernel restricted to the rows a call queries, the cell bias it
builds on the fly (time_bucket_dev), the page bookkeeping of hstu_pool_alloc_kernel / hstu_cache_append_kernel /
hstu_pool_release_kernel, and the host's extend_split.

The attention reference is hstu_block_reference.attention for the queried rows only: memory grows as [B, H, rows, keys], not as
[B, H, L, L], so a 16,384-item history can be checked row by row.  Where the kernels round is the same as there (e_x from the fp32
Q.K sum and the bias add, SILU_SLACK of the fast sigmoid, the bf16 pack U of A, the bf16 store of O), except the depth of the fp32
sum of A V: a row at cache position p sums p + 1 keys inside the CTAs of its splits and the combine then adds its
p // split + 1 split partials, so the per-term allowance is (p + 1 + splits of the row) ACC.
"""
import torch

from tests.attention_reference import U
from tests.dense_reference import ACC, C, SILU_SLACK
from tests.hstu_block_reference import _align, saved_layout

ATT_BLK = 64                    # keys per tile and query rows per CTA
POOL_ERR_RANGE, POOL_ERR_REPEAT = 1, 2


# ------------------------------------------------------------------------------------------------ host rule (csrc/api.cu)
def extend_split(B, n, H, capacity, sms):
    """keys per CTA: enough splits that B * H * ceil(n / 64) * splits reaches 4 CTAs per SM, rounded up to whole 64-key tiles"""
    base = B * H * -(-n // ATT_BLK)
    want = -(-4 * sms // base)
    per = -(-capacity // want)
    return -(-per // ATT_BLK) * ATT_BLK


def extend_nsplit(B, n, H, capacity, sms):
    return -(-capacity // extend_split(B, n, H, capacity, sms))


def extend_workspace_bytes(B, n, D, H, capacity, sms):
    """carve_extend: the forward's activation layout of the B * n chunk rows, then the [splits, B * n, D] fp32 partials"""
    T = B * n
    return saved_layout(T, D)["bytes"] + _align(extend_nsplit(B, n, H, capacity, sms) * T * D * 4)


# ------------------------------------------------------------------------------------------------ cell bias
def _floor_log2(d):
    """floor(log2 d) of int64 d >= 1, exact (the fp64 log2 of a value near 2^k may round across k)"""
    e = torch.floor(torch.log2(d.double())).long().clamp(0, 62)
    one = torch.ones_like(d)
    e = e - (torch.bitwise_left_shift(one, e) > d).long()
    up = (e < 62) & (torch.bitwise_left_shift(one, (e + 1).clamp_max(62)) <= d)
    return e + up.long()


def time_bucket(dt, thr, ntime):
    """time_bucket_dev: |dt| clamped at 1, floor(log2), + 1 at or above thr[e + 1], clamped to ntime - 1.  dt int64, thr [65]."""
    d = dt.abs().clamp_min(1)
    e = _floor_log2(d)
    thr = thr.to(d.device)
    return torch.minimum(e + (d >= thr[e + 1]).long(), torch.full_like(e, ntime - 1))


def cell_bias(pos, K, wpos, pos_bucket, wtime=None, tq=None, tk=None, thr=None, ntime=0):
    """The fp32 table sum att_build_table gives cell (row, key j < K): wpos[bucket] (+ wtime[time bucket]), one fp32 add.
    pos [B, R] cache position of each queried row (-1: none), wpos [npos, H] (the live row alone, [1, H], when pos_bucket is None:
    uniform buckets), pos_bucket [>= K] uint8 bucket of each delta p - j or None, wtime [ntime, H] or None (no time term) with
    tq [B, R] / tk [B, K] int64 timestamps and thr [65].  -> w [B, H, R, K] fp32 (junk where j > p)."""
    B, R = pos.shape
    j = torch.arange(K, device=pos.device)
    if pos_bucket is None:
        w = wpos.float()[0][None, :, None, None].expand(B, -1, R, K)
    else:
        delta = (pos[:, :, None].long() - j).clamp(0, pos_bucket.numel() - 1)
        w = wpos.float()[pos_bucket.to(pos.device).long()[delta]].permute(0, 3, 1, 2)
    if wtime is not None:
        tb = time_bucket(tq[:, :, None] - tk[:, None, :], thr, ntime)
        w = w + wtime.float()[tb].permute(0, 3, 1, 2)
    return w.contiguous()


# ------------------------------------------------------------------------------------------------ attention of the queried rows
def attention_rows(q, k, v, w, valid, depth, H):
    """q [B, R, D] bf16 queries, k / v [B, K, D] bf16 keys and values of each row's user, w [B, H, R, K] fp32 cell bias, valid
    [B, R, K] (key j <= the row's position), depth [B, R] or a number: terms of the fp32 A V sum.  -> "O" [B, R, D] with "a_O"."""
    B, R, D = q.shape
    dh = D // H
    qh = q.double().reshape(B, R, H, dh).transpose(1, 2)
    kh = k.double().reshape(B, -1, H, dh).transpose(1, 2)
    vh = v.double().reshape(B, -1, H, dh).transpose(1, 2)
    x = qh @ kh.transpose(-1, -2) + w.double()
    e_x = dh * ACC * (qh.abs() @ kh.abs().transpose(-1, -2)) + C * x.abs()
    ok = valid[:, None]
    zero = torch.zeros((), dtype=torch.float64, device=x.device)
    A = torch.where(ok, x * torch.sigmoid(x), zero)
    e_A = torch.where(ok, 1.1 * e_x + SILU_SLACK * x.abs() * (1 + x.abs()), zero)
    del x, e_x
    dep = torch.as_tensor(depth, dtype=torch.float64, device=A.device)
    if dep.dim() == 2:
        dep = dep[:, None, :, None]
    mA = e_A + (U + dep * ACC) * A.abs()
    del e_A
    O = A @ vh
    a_O = U * O.abs() + (1 + U) * (mA @ vh.abs())
    merge = lambda t: t.transpose(1, 2).reshape(B, R, D)                  # noqa: E731
    return {"O": merge(O), "a_O": merge(a_O)}


def row_depth(pos, split):
    """the fp32 summation depth of the row at cache position p: p + 1 keys and p // split + 1 split partials"""
    p = pos.clamp_min(0)
    return p + 1 + p // split + 1


# ------------------------------------------------------------------------------------------------ page bookkeeping
def _pages(items, ps):
    return -(-items // ps)


def pool_alloc(users, counts, lengths, page_table, free_stack, free_top, max_users, max_items, page_size):
    """hstu_pool_alloc_kernel on plain integers.  users [B], counts [B] valid items of each row, lengths [max_users],
    page_table [max_users, pt_ld], free_stack [num_pages], free_top: int.  Rows in order: a row is accepted when its user is in
    range and no earlier row names it; it needs ceil(min(len + count, max_items) / ps) - ceil(len / ps) pages, taken from the top of
    the free stack starting after what the earlier rows ASKED for.  -> page_table (new), room [B] (-1 rejected), free_top, errors."""
    users, counts, lengths = users.tolist(), counts.tolist(), lengths.tolist()
    pt = page_table.clone()
    stack = free_stack.tolist()
    avail = int(free_top)
    seen, room, handed, err = set(), [], 0, 0
    for u, cnt in zip(users, counts):
        if not 0 <= u < max_users:
            err |= POOL_ERR_RANGE
            room.append(-1)
            continue
        if u in seen:
            err |= POOL_ERR_REPEAT
            room.append(-1)
            continue
        seen.add(u)
        l = lengths[u]
        have = _pages(l, page_size)
        need = max(0, _pages(min(l + cnt, max_items), page_size) - have)
        got = max(0, min(need, avail - handed))
        for k in range(got):
            pt[u, have + k] = stack[avail - 1 - (handed + k)]
        room.append(min(max_items, (have + got) * page_size))
        handed += need
    return {"page_table": pt, "room": torch.tensor(room, dtype=torch.int32), "free_top": avail - min(handed, avail), "errors": err}


def cache_append(ids, ts, users, room, lengths, overflow, cap):
    """hstu_cache_append_kernel on plain integers.  ids / ts [B, n] (ts None: 0 stored), users [B] (None: row b is user b), room [B]
    (None: cap for every row).  -> positions [B, n] int32, last_row [B] int32, lengths, overflow (new) and writes: a list of
    (user, position, timestamp) the kernel stores."""
    B, n = ids.shape
    L, ov = lengths.clone(), overflow.clone()
    positions = torch.full((B, n), -1, dtype=torch.int32)
    last_row = torch.full((B,), -1, dtype=torch.int32)
    writes = []
    valid = (ids != 0).tolist()
    for b in range(B):
        lim = cap if room is None else int(room[b])
        if lim < 0:
            continue
        u = b if users is None else int(users[b])
        base, count = int(L[u]), 0
        for r in range(n):
            if not valid[b][r]:
                continue
            q = base + count
            if q < lim:
                positions[b, r] = q
                writes.append((u, q, 0 if ts is None else int(ts[b, r])))
            count += 1
            last_row[b] = r
        total = base + count
        L[u] = min(total, lim)
        if total > lim:
            ov[u] = 1
    return {"positions": positions, "last_row": last_row, "lengths": L, "overflow": ov, "writes": writes}


def pool_release(users, lengths, overflow, page_table, free_stack, free_top, max_users, num_pages, page_size):
    """hstu_pool_release_kernel on plain integers: each accepted row's pages go back onto the free stack in row order, then page
    order; the user's length and overflow flag become 0.  -> free_stack, free_top, lengths, overflow, errors, released users."""
    stack = free_stack.clone()
    L, ov = lengths.clone(), overflow.clone()
    top, pushed, err, seen = int(free_top), 0, 0, []
    for u in users.tolist():
        if not 0 <= u < max_users:
            err |= POOL_ERR_RANGE
            continue
        if u in seen:
            err |= POOL_ERR_REPEAT
            continue
        seen.append(u)
        pages = _pages(int(L[u]), page_size)
        for k in range(pages):
            if top + pushed + k < num_pages:
                stack[top + pushed + k] = page_table[u, k]
        L[u], ov[u] = 0, 0
        pushed += pages
    return {"free_stack": stack, "free_top": min(top + pushed, num_pages), "lengths": L, "overflow": ov, "errors": err,
            "released": seen}


def cache_rows(users, lengths, K, page_table=None, page_size=None, cap=None):
    """[B, K] int64 row of item j of each call row's user in the [pages * page_size] (pool) or [users * cap] (dense) rows of K | V
    and timestamps, and the [B, K] mask j < length.  users [B] (None: row b is user b), lengths [B] of the rows' users."""
    j = torch.arange(K, device=lengths.device)
    ok = j[None, :] < lengths[:, None]
    if users is None:
        users = torch.arange(lengths.shape[0])
    if page_table is None:
        rows = users.to(lengths.device).long()[:, None] * cap + j[None, :]
    else:
        jj = torch.where(ok, j[None, :], torch.zeros_like(j)[None, :])
        pages = page_table.long()[users.long()[:, None], jj // page_size]
        rows = pages * page_size + jj % page_size
    return torch.where(ok, rows, torch.zeros_like(rows)), ok
