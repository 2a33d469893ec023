"""Cached incremental HSTU inference (HSTU.new_state / HSTU.extend) against the fp64 oracle and the full-recompute last_logits."""
import pytest
import torch

from tests.sign_fixed_buckets import use_sign_fixed_oracle
from tests.util import budget, make_batch, relerr

pytestmark = pytest.mark.gpu

V, NB = 500, 2


def _model(D, H, use_time=True, seed=0, dropout=0.0):
    from genrec_b200.hstu import HSTU
    torch.manual_seed(seed)
    m = HSTU(V, 64, D, H, NB, dropout=dropout, use_temporal_bias=use_time)
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "attention_bias" in n:
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
    return m.to("cuda").eval()


def _oracle_last(m, ids, ts):
    from oracle import hstu as oh
    sd = {k: v.detach().double().cpu() for k, v in m.state_dict().items()}
    logits, _ = oh.hstu_forward(ids.cpu(), ts.cpu() if ts is not None else None, None, sd, m.layers[0].num_heads, len(m.layers),
                                use_temporal_bias=m.use_temporal_bias)
    return logits[:, -1]


def _check(ext, m, ids, ts, rows):
    """extend's logits of `rows` are as close to the fp64 oracle as last_logits on the same left-padded batch."""
    ref = _oracle_last(m, ids, ts)
    full = m.last_logits(ids, ts)
    e, b = relerr(ext[rows], ref[rows]), budget(full[rows], ref[rows])
    assert e <= b, (e, b)
    return full


def _sign_fixed(m):
    """Set the sign-fixed (non-uniform) position-bucket table through bucket_of_delta: bucket(i - j) instead of bucket(j - i)."""
    for layer in m.layers:
        rpb = layer.position_bias
        rpb._relative_position_bucket = (lambda f: (lambda rel: f(-rel)))(rpb._relative_position_bucket)
        rpb._table_cache.clear()
        rpb._uniform_cache.clear()


@pytest.mark.parametrize("D,H", [(64, 2), (128, 4), (128, 2), (256, 8)])
@pytest.mark.parametrize("time_mode", ["time", "no_temporal_bias", "timestamps_none"])
def test_prefill_matches_full_forward(D, H, time_mode):
    m = _model(D, H, use_time=time_mode != "no_temporal_bias")
    ids, ts, _ = make_batch(4, 50, V, seed=D + H)
    ids, ts = ids.cuda(), ts.cuda()
    if time_mode == "timestamps_none":
        ts = None
    st = m.new_state(4, 64)
    ext = m.extend(st, ids, ts)
    assert ext.shape == (4, V + 1) and torch.isfinite(ext).all()
    _check(ext, m, ids, ts, [0, 1, 3])                  # row 2 is all padding
    assert st.lengths.tolist() == [50, 50 - 50 // 3, 0, 50]


def _chunks(B, widths, seed, max_pad=3):
    """Per chunk of width w, user b's row holds min(b * max_pad, w - 1) left pads and then its next items."""
    g = torch.Generator().manual_seed(seed)
    chunks = []
    for w in widths:
        ids = torch.randint(1, V + 1, (B, w), generator=g)
        ts = torch.randint(1, 3 * 86400, (B, w), generator=g)
        ts[:, ::3] = torch.randint(0, 30, (B, (w + 2) // 3), generator=g)
        for b in range(B):
            p = min(b * max_pad, w - 1)
            ids[b, :p] = 0
        chunks.append((ids, ts))
    return chunks


def _concat(chunks, upto):
    """left-padded [B, Lmax] batch of each user's items in the first `upto` chunks (timestamps made increasing per user)."""
    B = chunks[0][0].shape[0]
    rows_i, rows_t = [], []
    for b in range(B):
        items = torch.cat([c[0][b] for c in chunks[:upto]])
        gaps = torch.cat([c[1][b] for c in chunks[:upto]])
        keep = items != 0
        rows_i.append(items[keep])
        rows_t.append(gaps[keep])
    Lm = max(len(r) for r in rows_i)
    ids = torch.zeros(B, Lm, dtype=torch.int64)
    ts = torch.zeros(B, Lm, dtype=torch.int64)
    for b in range(B):
        n = len(rows_i[b])
        ids[b, Lm - n:] = rows_i[b]
        ts[b, Lm - n:] = rows_t[b]
    return ids, ts


def _absolute_ts(chunks):
    """turn the per-slot gaps into increasing timestamps per user, identically in chunk and concatenated form"""
    B = chunks[0][0].shape[0]
    last = torch.full((B,), 1_300_000_000, dtype=torch.int64)
    out = []
    for ids, gaps in chunks:
        ts = last[:, None] + torch.cumsum(gaps * (ids != 0), 1)
        ts[ids == 0] = 0
        last = torch.where((ids != 0).any(1), ts.max(1).values, last)
        out.append((ids, ts))
    return out


def _run_chunked(m, B, widths, seed):
    chunks = _absolute_ts(_chunks(B, widths, seed))
    st = m.new_state(B, sum(widths))
    for k, (ids, ts) in enumerate(chunks):
        ext = m.extend(st, ids.cuda(), ts.cuda())
        cids, cts = _concat(chunks, k + 1)
        _check(ext, m, cids.cuda(), cts.cuda(), list(range(B)))
    assert st.lengths.cpu().tolist() == [int((_concat(chunks, len(chunks))[0][b] != 0).sum()) for b in range(B)]
    assert not st.overflowed().any()


@pytest.mark.parametrize("B,widths,D,H", [(3, [1, 7, 64, 65, 63], 64, 2), (3, [1, 7, 64, 65, 63], 128, 4),
                                          (1, [1, 7, 64, 65, 1000], 64, 2)])
def test_chunked_matches_full_forward(B, widths, D, H):
    _run_chunked(_model(D, H), B, widths, seed=B + D)


def test_non_uniform_position_buckets_left_padded_chunks(monkeypatch):
    m = _model(64, 2, seed=7)
    _sign_fixed(m)
    use_sign_fixed_oracle(monkeypatch)
    assert not m.layers[0].position_bias.uniform_of(200, "cuda")[0]
    _run_chunked(m, 3, [1, 7, 64, 65, 63], seed=11)


def _state_tensors(st):
    return [st.kv, st.timestamps, st.lengths, st.overflow, st.last_hidden]


def test_all_pad_row_keeps_state_and_logits():
    m = _model(128, 4)
    ids, ts, _ = make_batch(4, 30, V, seed=2)
    ids, ts = ids.cuda(), ts.cuda()
    st = m.new_state(4, 64)
    first = m.extend(st, ids, ts)
    before = [t.clone() for t in _state_tensors(st)]
    nid = torch.randint(1, V + 1, (4, 5), device="cuda")
    nts = ts[:, -1:] + torch.arange(1, 6, device="cuda")
    nid[1] = 0
    nts[1] = 0
    second = m.extend(st, nid, nts)
    assert torch.equal(second[1], first[1])
    for a, b in zip(_state_tensors(st), before):
        assert torch.equal(a[:, 1] if a.dim() == 4 else a[1], b[:, 1] if b.dim() == 4 else b[1])
    assert not torch.equal(second[0], first[0])


def test_refusals():
    from genrec_b200 import _lib
    m = _model(64, 2)
    ids, ts, _ = make_batch(2, 8, V, seed=3, pad=False)
    ids, ts = ids.cuda(), ts.cuda()
    st = m.new_state(2, 10)
    m.extend(st, ids, ts)
    n0 = _lib.launches()
    with pytest.raises(ValueError, match="capacity"):
        m.extend(st, ids[:, :3], ts[:, :3])
    assert _lib.launches() == n0                        # refused before any launch
    # stale state: a torch optimizer step, then load_state_dict
    for p in m.parameters():
        p.grad = torch.ones_like(p)
    torch.optim.Adam(m.parameters(), lr=1e-3).step()
    with pytest.raises(RuntimeError, match="rebuild"):
        m.extend(st, ids[:, :1], ts[:, :1])
    st = m.new_state(2, 10)
    m.extend(st, ids, ts)
    m.load_state_dict(_model(64, 2, seed=9).state_dict())
    with pytest.raises(RuntimeError, match="rebuild"):
        m.extend(st, ids[:, :1], ts[:, :1])
    # training mode with dropout, fp32 precision
    md = _model(64, 2, dropout=0.2).train()
    with pytest.raises(RuntimeError, match="dropout"):
        md.extend(md.new_state(2, 10), ids, ts)
    m.set_precision("fp32")
    with pytest.raises(RuntimeError, match="bf16"):
        m.extend(m.new_state(2, 10), ids, ts)


def _prefilled(m, lens, width, cap, seed):
    g = torch.Generator().manual_seed(seed)
    B = len(lens)
    ids = torch.randint(1, V + 1, (B, width), generator=g)
    ts = 1_300_000_000 + torch.cumsum(torch.randint(1, 86400, (B, width), generator=g), 1)
    for b, n in enumerate(lens):
        ids[b, :width - n] = 0
        ts[b, :width - n] = 0
    st = m.new_state(B, cap)
    m.extend(st, ids.cuda(), ts.cuda())
    return st, ids.cuda(), ts.cuda()


def test_deterministic():
    m = _model(128, 4)
    runs = []
    for _ in range(2):
        st, ids, ts = _prefilled(m, [150, 90, 3], 150, 256, seed=4)
        out = m.extend(st, ids[:, -2:], ts[:, -2:] + 1000)
        runs.append((out, _state_tensors(st)))
    assert torch.equal(runs[0][0], runs[1][0])
    for a, b in zip(runs[0][1], runs[1][1]):
        assert torch.equal(a, b)


def test_cuda_graph_replay_and_overflow():
    m = _model(128, 4)
    cap = 20
    eager, _, _ = _prefilled(m, [18, 10, 5], 18, cap, seed=5)
    graphed, _, _ = _prefilled(m, [18, 10, 5], 18, cap, seed=5)
    chunk_ids = torch.tensor([[11], [12], [0]], device="cuda")
    chunk_ts = torch.tensor([[1_400_000_000], [1_400_000_000], [0]], device="cuda")
    static_ids, static_ts = chunk_ids.clone(), chunk_ts.clone()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = m.extend(graphed, static_ids, static_ts)
    for _ in range(2):                                  # eager and replayed extends agree bit for bit
        ref = m.extend(eager, chunk_ids, chunk_ts)
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, ref)
        for a, b in zip(_state_tensors(graphed), _state_tensors(eager)):
            assert torch.equal(a, b)
    with pytest.raises(ValueError, match="capacity"):  # the eager state is full: the host check refuses
        m.extend(eager, chunk_ids, chunk_ts)
    for _ in range(2):                                  # replays past capacity: user 0's items are dropped and flagged
        g.replay()
    torch.cuda.synchronize()
    assert graphed.overflowed().tolist() == [True, False, False]
    assert graphed.lengths.tolist() == [cap, 14, 5]
    assert torch.equal(graphed.kv[:, 0], eager.kv[:, 0]) and torch.equal(graphed.timestamps[0], eager.timestamps[0])
    # a later extend of a user with room is unaffected by the overflow of another
    late_ids = torch.tensor([[0], [0], [13]], device="cuda")
    late_ts = torch.tensor([[0], [0], [1_400_000_100]], device="cuda")
    fresh, _, _ = _prefilled(m, [18, 10, 5], 18, cap, seed=5)
    a = m.extend(graphed, late_ids, late_ts)
    b = m.extend(fresh, late_ids, late_ts)
    assert torch.equal(a[2], b[2])
    assert torch.equal(graphed.kv[:, 2], fresh.kv[:, 2]) and graphed.lengths[2].item() == 6
