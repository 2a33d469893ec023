"""Integer restatement of the packed (jagged) chunk bookkeeping of csrc/attn_hstu_extend.cuh, built on tests/extend_reference.py:
hstu_cache_append_kernel<true> and hstu_pool_alloc_kernel<true> on a chunk of T token rows with offsets [B+1] and max_len.

Sequence b is the token rows seq_span(offsets, T, max_len, b) (common.cuh): offsets clamped to [0, T], non-decreasing, and the
length cut at max_len.  Rows in no sequence are idle.  Each sequence is handled as the row of a padded [B, max_len] chunk that
holds the same ids in the same order, so the packed functions here map a packed chunk to that padded chunk, run the padded
reference, and map the results back to token rows.
"""
import torch

from tests import extend_reference as er


def seq_spans(offsets, T, max_len):
    """[(tok0, len)] of every sequence, clamped as seq_span clamps a device offsets."""
    o = [int(v) for v in offsets]
    spans = []
    for b in range(len(o) - 1):
        lo = min(max(o[b], 0), T)
        hi = min(max(o[b + 1], lo), T)
        spans.append((lo, min(hi - lo, max_len)))
    return spans


def to_padded(ids, ts, offsets, max_len):
    """The left-padded [B, max_len] chunk of a packed one (pads 0, their timestamps 0), and slot[t] = (b, column) of token row t
    (None for an idle row)."""
    T = ids.numel()
    spans = seq_spans(offsets, T, max_len)
    pids = torch.zeros(len(spans), max_len, dtype=torch.int64)
    pts = torch.zeros(len(spans), max_len, dtype=torch.int64)
    slot = [None] * T
    for b, (t0, n) in enumerate(spans):
        c0 = max_len - n
        pids[b, c0:] = ids[t0:t0 + n]
        if ts is not None:
            pts[b, c0:] = ts[t0:t0 + n]
        for i in range(n):
            slot[t0 + i] = (b, c0 + i)
    return pids, (pts if ts is not None else None), slot


def packed_counts(ids, offsets, max_len):
    """[B] valid items (id != 0) of every sequence: what hstu_pool_alloc_kernel<true> counts."""
    spans = seq_spans(offsets, ids.numel(), max_len)
    return torch.tensor([int((ids[t0:t0 + n] != 0).sum()) for t0, n in spans], dtype=torch.int64)


def cache_append_packed(ids, ts, offsets, max_len, users, room, lengths, overflow, cap):
    """hstu_cache_append_kernel<true> restated row by row: positions [T] int32 (-1 for pads, dropped items and idle rows) and
    last_row [B] int32 holding the token row of each user's last valid item (-1: none), plus lengths / overflow / writes as
    extend_reference.cache_append returns them."""
    T = ids.numel()
    L, ov = lengths.clone(), overflow.clone()
    positions = torch.full((T,), -1, dtype=torch.int32)
    last_row = torch.full((len(offsets) - 1,), -1, dtype=torch.int32)
    writes = []
    for b, (t0, n) in enumerate(seq_spans(offsets, T, max_len)):
        lim = cap if room is None else int(room[b])
        if lim < 0:
            continue
        u = b if users is None else int(users[b])
        base, count = int(L[u]), 0
        for t in range(t0, t0 + n):
            if int(ids[t]) == 0:
                continue
            q = base + count
            if q < lim:
                positions[t] = q
                writes.append((u, q, 0 if ts is None else int(ts[t])))
            count += 1
            last_row[b] = t
        total = base + count
        L[u] = min(total, lim)
        if total > lim:
            ov[u] = 1
    return {"positions": positions, "last_row": last_row, "lengths": L, "overflow": ov, "writes": writes}


def padded_equivalent(ids, ts, offsets, max_len, users, room, lengths, overflow, cap):
    """extend_reference.cache_append on to_padded's chunk, with its positions and last_row mapped back to token rows: what the
    packed append must return."""
    pids, pts, slot = to_padded(ids, ts, offsets, max_len)
    ref = er.cache_append(pids, pts, users, room, lengths, overflow, cap)
    positions = torch.full((ids.numel(),), -1, dtype=torch.int32)
    for t, s in enumerate(slot):
        if s is not None:
            positions[t] = ref["positions"][s[0], s[1]]
    spans = seq_spans(offsets, ids.numel(), max_len)
    last_row = torch.tensor([-1 if int(r) < 0 else spans[b][0] + int(r) - (max_len - spans[b][1])
                             for b, r in enumerate(ref["last_row"])], dtype=torch.int32)
    return dict(ref, positions=positions, last_row=last_row)


def random_packed_chunk(g, B, max_len, V, idle=0, lengths=None, zero_frac=0.1):
    """A packed chunk of B sequences with lengths in [0, max_len] (or `lengths`), a few ids 0 inside sequences, and `idle` idle
    rows after them holding non-zero ids and timestamps.  -> ids [T], ts [T], offsets [B+1] (CPU int64)."""
    if lengths is None:
        lengths = torch.randint(0, max_len + 1, (B,), generator=g).tolist()
    offsets = torch.tensor([0] + torch.tensor(lengths).cumsum(0).tolist(), dtype=torch.int64)
    T = int(offsets[-1]) + idle
    ids = torch.randint(1, V + 1, (max(T, 1),), generator=g)
    ids[torch.rand(ids.shape, generator=g) < zero_frac] = 0
    if T > idle:
        ids[T - idle:] = torch.randint(1, V + 1, (idle,), generator=g)
    ts = 1_300_000_000 + torch.cumsum(torch.randint(1, 10 ** 5, ids.shape, generator=g), 0)
    return ids, ts, offsets
