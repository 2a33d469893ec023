"""The references of tests/extend_reference.py against the ones they restate (no GPU): the row-restricted attention against
hstu_block_reference.attention, the cell bias against hstu_block_reference.cell_bias on an index matrix built from the oracle's
bucket rules, the integer time bucket against the oracle's fp32 expression, the pool bookkeeping on hand-made cases, and the
restated extend_split against the library's workspace query."""
import ctypes

import pytest
import torch

from tests import extend_reference as er
from tests import hstu_block_reference as hr


@pytest.fixture(scope="module")
def lib():
    from genrec_b200 import build
    build.build()
    from genrec_b200 import _lib
    return _lib.load()


# ------------------------------------------------------------------------------------------------ attention of the queried rows
@pytest.mark.parametrize("L,D,H", [(1, 64, 2), (70, 128, 4), (130, 128, 2)])
def test_attention_rows_equal_full_attention_rows(L, D, H):
    g = torch.Generator().manual_seed(L + D)
    B = 3
    P = (torch.randn(B, L, 4 * D, generator=g) * 0.8).bfloat16()
    w = (0.3 * torch.randn(B, H, L, L, generator=g)).float()
    pad = torch.zeros(B, L, dtype=torch.bool)
    pad[1, : L // 3] = True
    pad[2, L // 2] = True
    valid = hr.causal_valid(pad)
    full = hr.attention(P, w, valid, H)
    rows = torch.tensor(sorted({0, L // 2, L - 1, max(0, L - 2)}))
    Vc, Qc, Kc = P[..., D:2 * D], P[..., 2 * D:3 * D], P[..., 3 * D:]
    got = er.attention_rows(Qc[:, rows], Kc, Vc, w[:, :, rows], valid[:, 0, rows], L, H)
    for name in ("O", "a_O"):
        torch.testing.assert_close(got[name], full[name][:, rows], rtol=1e-12, atol=1e-14)


def test_row_depth():
    pos = torch.tensor([[0, 63, 64, 703, 704, 2047, -1]])
    assert er.row_depth(pos, 704).tolist() == [[2, 65, 66, 705, 707, 2051, 2]]


# ------------------------------------------------------------------------------------------------ cell bias
def _edge_dts():
    big = [(1 << k) + d for k in range(63) for d in (-1, 0, 1)] + [(1 << 63) - 1, 1023, 1024, 0]
    return torch.tensor([v for v in big if v < (1 << 63)] + [-v for v in big if 0 < v < (1 << 63)], dtype=torch.int64)


@pytest.mark.parametrize("ntime", [1, 20, 64])
def test_time_bucket_matches_the_oracle_expression(ntime):
    from genrec_b200.hstu import time_bucket_thresholds
    from oracle import hstu as oh
    thr = time_bucket_thresholds()
    g = torch.Generator().manual_seed(ntime)
    dt = torch.cat([_edge_dts(), torch.randint(-(1 << 40), 1 << 40, (4000,), generator=g),
                    torch.randint(-(1 << 62), 1 << 62, (4000,), generator=g)])
    assert torch.equal(er.time_bucket(dt, thr, ntime), oh.temporal_bucket(dt, ntime))


@pytest.mark.parametrize("uniform", [True, False])
@pytest.mark.parametrize("timed", [True, False])
def test_cell_bias_matches_the_index_matrix_decode(uniform, timed):
    """er.cell_bias of every row of a full history equals hr.cell_bias of the index matrix built from the oracle's bucket rules"""
    from genrec_b200.hstu import time_bucket_thresholds
    from oracle import hstu as oh
    L, H, npos, md, ntime = 150, 2, 32, 100, 20
    g = torch.Generator().manual_seed(7)
    ts = 1_300_000_000 + torch.cumsum(torch.randint(0, 3 * 86400, (2, L), generator=g), 1)
    ts[1] = torch.arange(L) * (1 << 50)
    wpos = 0.3 * torch.randn(npos, H, generator=g)
    wtime = 0.5 * torch.randn(ntime, H, generator=g) if timed else None
    i = torch.arange(L)
    delta = i[:, None] - i[None, :]
    pb = torch.full((L, L), 5) if uniform else oh.position_bucket(delta, npos, md)
    tb = oh.temporal_bucket(ts[:, :, None] - ts[:, None, :], ntime) if timed else torch.zeros(2, L, L, dtype=torch.int64)
    idx = torch.where(delta >= 0, pb * 64 + tb, torch.full_like(tb, (1 if uniform else npos) * 64))
    live = wpos[5:6] if uniform else wpos
    want, masked, _, _ = hr.cell_bias(idx.to(torch.int16), live, wtime, 1 if uniform else npos, H)
    pos_bucket = None if uniform else oh.position_bucket(i, npos, md).to(torch.uint8)
    got = er.cell_bias(i[None].expand(2, L), L, live, pos_bucket, wtime, ts, ts, time_bucket_thresholds(), ntime)
    causal = ~masked.expand_as(want)
    assert torch.equal(got[causal], want[causal])


# ------------------------------------------------------------------------------------------------ page bookkeeping
def _hand_pool():
    """4 users, pages of 64 items, max_items 256; users 1 and 3 hold 60 and 130 items; pages 10..14 free, 14 on top"""
    pt = torch.full((4, 4), -1, dtype=torch.int32)
    pt[1, 0] = 7
    pt[3, :3] = torch.tensor([8, 9, 6])
    stack = torch.tensor([10, 11, 12, 13, 14, 99, 99, 99, 99, 99], dtype=torch.int32)
    return dict(lengths=torch.tensor([0, 60, 0, 130], dtype=torch.int32), page_table=pt, free_stack=stack, free_top=5)


def test_pool_alloc_hand_made():
    p = _hand_pool()
    users = torch.tensor([1, 3, 1, 7, 0, 2])
    counts = torch.tensor([10, 100, 5, 3, 200, 64])
    r = er.pool_alloc(users, counts, p["lengths"], p["page_table"], p["free_stack"], p["free_top"], 4, 256, 64)
    # row 0: 60 -> 70 items, one page more (14) ; row 1: 130 -> 230, page 13 ; row 2 repeats user 1 ; row 3 is out of range ;
    # row 4: 0 -> 200 items wants 4 pages, finds 3 (12, 11, 10) ; row 5 finds the stack empty
    assert r["room"].tolist() == [128, 256, -1, -1, 192, 0]
    assert r["errors"] == er.POOL_ERR_RANGE | er.POOL_ERR_REPEAT
    assert r["free_top"] == 0
    assert r["page_table"][1, :2].tolist() == [7, 14] and r["page_table"][3].tolist() == [8, 9, 6, 13]
    assert r["page_table"][0, :3].tolist() == [12, 11, 10] and r["page_table"][2].tolist() == [-1] * 4
    # the append: user 0's items beyond its 192 are dropped and flag it; the rejected rows write nothing
    ids = torch.zeros(6, 200, dtype=torch.int64)
    for b, c in enumerate(counts.tolist()):
        ids[b, 200 - c:] = 1
    ids[0, 195] = 0                                  # a pad inside a row: positions count items
    a = er.cache_append(ids, None, users, r["room"], p["lengths"], torch.zeros(4, dtype=torch.uint8), 256)
    assert a["lengths"].tolist() == [192, 69, 0, 230] and a["overflow"].tolist() == [1, 0, 1, 0]     # user 2 found no page
    assert a["positions"][0, 190:].tolist() == [60, 61, 62, 63, 64, -1, 65, 66, 67, 68]
    assert a["positions"][4, :192].tolist() == list(range(192)) and bool((a["positions"][4, 192:] == -1).all())
    assert bool((a["positions"][2:4] == -1).all()) and bool((a["positions"][5] == -1).all())
    assert a["last_row"].tolist() == [199, 199, -1, -1, 199, 199]
    assert {(u, q) for u, q, _ in a["writes"]} == ({(1, q) for q in range(60, 69)} | {(3, q) for q in range(130, 230)} |
                                                  {(0, q) for q in range(192)})


def test_pool_release_hand_made():
    p = _hand_pool()
    r = er.pool_release(torch.tensor([3, 5, 1, 3, 0]), p["lengths"], torch.tensor([0, 1, 0, 1], dtype=torch.uint8), p["page_table"],
                        p["free_stack"], p["free_top"], 4, 10, 64)
    assert r["free_stack"].tolist() == [10, 11, 12, 13, 14, 8, 9, 6, 7, 99]     # user 3's pages in page order, then user 1's
    assert r["free_top"] == 9 and r["errors"] == er.POOL_ERR_RANGE | er.POOL_ERR_REPEAT
    assert r["lengths"].tolist() == [0, 0, 0, 0] and r["overflow"].tolist() == [0, 0, 0, 0] and r["released"] == [3, 1, 0]


# ------------------------------------------------------------------------------------------------ extend_split
# (B, n, D, H, capacity) -> (split, splits) at 132 SMs: the regimes tests/test_hstu_extend_exact_gpu.py runs
REGIMES = [((132, 1, 128, 4, 2048), (2048, 1)), ((32, 1, 256, 8, 2048), (704, 3)), ((128, 1, 128, 4, 200), (128, 2)),
           ((64, 1, 256, 4, 1000), (384, 3)), ((40, 65, 128, 4, 700), (384, 2)), ((1, 64, 128, 2, 16384), (64, 256)),
           ((1, 16384, 128, 2, 16384), (8192, 2)), ((1100, 1, 64, 2, 192), (192, 1))]


def test_extend_split_regimes_at_132_sms():
    for (B, n, D, H, cap), want in REGIMES:
        assert (er.extend_split(B, n, H, cap, 132), er.extend_nsplit(B, n, H, cap, 132)) == want, (B, n, D, H, cap)


def test_extend_split_matches_the_library(lib):
    from genrec_b200._lib import HstuDims
    shapes = [s for s, _ in REGIMES] + [(B, n, D, H, cap) for B in (1, 3, 33, 528, 2000) for n in (1, 63, 65, 200)
                                        for D, H in ((64, 2), (256, 4)) for cap in (1, 64, 65, 1000, 16384)]
    for B, n, D, H, cap in shapes:
        d = HstuDims(B, n, D, H, 32, 64, 0.0, 0, None, 0)
        assert lib.grb_hstu_layer_extend_workspace_bytes(ctypes.byref(d), cap) == er.extend_workspace_bytes(B, n, D, H, cap, 132), \
            (B, n, D, H, cap)
