"""Packed (jagged) chunks for the cached extend without a GPU: the refusals of HSTU.extend_jagged / extend_users_jagged before any
launch, the host bound of a pool for per-user lengths, the integer restatement of the packed append and allocation against the
padded references of tests/extend_reference.py, and the new entry points in the header and the ctypes binding."""
import os
import re

import pytest
import torch

from tests import extend_jagged_reference as jr
from tests import extend_reference as er

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["grb_hstu_cache_append_jagged", "grb_hstu_pool_append_jagged", "grb_hstu_layer_extend_workspace_bytes_jagged",
               "grb_hstu_layer_extend_jagged", "grb_hstu_layer_extend_paged_workspace_bytes_jagged", "grb_hstu_layer_extend_paged_jagged"]


def _model():
    from genrec_b200.hstu import HSTU
    torch.manual_seed(0)
    return HSTU(50, 80, 64, 2, 1, dropout=0.0).eval()


def _ids(T):
    return torch.randint(1, 51, (T,), dtype=torch.int64)


@pytest.mark.parametrize("bad, msg", [
    ("offsets_first", "offsets\\[0\\] must be 0"),
    ("offsets_decrease", "non-decreasing"),
    ("longer_than_max_len", "exceeds max_len"),
    ("offsets_past_T", "exceeds the 6 token rows"),
    ("batch_size", "one sequence per user"),
    ("ts_shape", "timestamps must be \\[6\\]"),
    ("max_len_capacity", "exceeds the state's capacity|exceeds the pool's max_items"),
    ("topk_and_candidates", "not both"),
    ("exclude_alone", "exclude needs top_k or num_candidates"),
    ("max_len0", "max_len must be an int"),
])
@pytest.mark.parametrize("target", ["state", "pool"])
def test_refusals_before_any_launch(bad, msg, target):
    """Every refusal is a ValueError raised on the host; none needs a device (the tensors here are on the CPU)."""
    m = _model()
    ids, off, max_len, ts, kw = _ids(6), torch.tensor([0, 2, 6]), 4, None, {}
    if bad == "offsets_first":
        off = torch.tensor([1, 2, 6])
    elif bad == "offsets_decrease":
        off = torch.tensor([0, 3, 2])
    elif bad == "longer_than_max_len":
        off = torch.tensor([0, 1, 6])
    elif bad == "offsets_past_T":
        off, max_len = torch.tensor([0, 2, 7]), 5
    elif bad == "batch_size":
        off = torch.tensor([0, 2, 4, 6])
    elif bad == "ts_shape":
        ts = torch.zeros(2, 3, dtype=torch.int64)
    elif bad == "max_len_capacity":
        max_len = 9
    elif bad == "topk_and_candidates":
        kw = dict(top_k=5, num_candidates=10)
    elif bad == "exclude_alone":
        kw = dict(exclude=torch.zeros(2, 1, dtype=torch.int64))
    else:
        max_len = 0
    with pytest.raises(ValueError, match=msg):
        if target == "state":
            m.extend_jagged(m.new_state(2, 8), ids, off, max_len, ts, **kw)
        else:
            m.extend_users_jagged(m.new_pool(4, 4, 64, 8), torch.tensor([0, 3]), ids, off, max_len, ts, **kw)


def test_refuses_fp32_and_training_mode():
    m = _model().set_precision("fp32")
    with pytest.raises(RuntimeError, match="bf16"):
        m.extend_jagged(m.new_state(2, 8), _ids(6), torch.tensor([0, 2, 6]), 4)
    m = _model().set_precision("bf16")
    m.layers[0].dropout.p = 0.1
    m.train()
    with pytest.raises(RuntimeError, match="dropout"):
        m.extend_users_jagged(m.new_pool(4, 4, 64, 8), [0, 1], _ids(6), torch.tensor([0, 2, 6]), 4)


def test_pool_bound_advances_by_each_users_length():
    """HSTUPool._check_room with the per-user lengths of a packed chunk: each user's bound moves by their own length, and the
    page bound by the pages those lengths need."""
    from genrec_b200.hstu import HSTUPool
    pool = HSTUPool(8, 10, 64, 256, 1, 64, "cpu")
    pool.items_bound[torch.tensor([1, 5])] = torch.tensor([60, 10])
    pool.pages_bound = 2
    u = torch.tensor([1, 5, 2])
    new, pages = pool._check_room(u, torch.tensor([10, 0, 129]))
    assert new.tolist() == [70, 10, 129]
    assert pages == 2 + 1 + 0 + 3
    with pytest.raises(ValueError, match="max_items"):
        pool._check_room(u, torch.tensor([197, 0, 0]))


def _check_against_padded(g, B, max_len, idle, pool_users, cap, lengths=None, room_rule=None):
    V = 40
    ids, ts, off = jr.random_packed_chunk(g, B, max_len, V, idle=idle, lengths=lengths)
    nu = (max(pool_users) + 1) if pool_users is not None else B
    L0 = torch.randint(0, cap, (nu,), generator=g).int()
    ov0 = torch.zeros(nu, dtype=torch.uint8)
    users = torch.tensor(pool_users) if pool_users is not None else None
    room = None
    if room_rule is not None:
        room = torch.tensor([room_rule(b) for b in range(B)], dtype=torch.int32)
    got = jr.cache_append_packed(ids, ts, off, max_len, users, room, L0, ov0, cap)
    want = jr.padded_equivalent(ids, ts, off, max_len, users, room, L0, ov0, cap)
    for k in ("positions", "last_row", "lengths", "overflow"):
        assert torch.equal(got[k], want[k]), k
    assert got["writes"] == want["writes"]
    # idle rows never get a position; last_row names an item of its own sequence
    spans = jr.seq_spans(off, ids.numel(), max_len)
    inside = torch.zeros(ids.numel(), dtype=torch.bool)
    for t0, n in spans:
        inside[t0:t0 + n] = True
    assert bool((got["positions"][~inside] == -1).all())
    for b, r in enumerate(got["last_row"].tolist()):
        assert r == -1 or (spans[b][0] <= r < spans[b][0] + spans[b][1] and int(ids[r]) != 0)
    # the allocation counts the same items as the padded chunk's rows
    pids, _, _ = jr.to_padded(ids, ts, off, max_len)
    assert torch.equal(jr.packed_counts(ids, off, max_len), (pids != 0).sum(1))
    if pool_users is not None:
        pt = torch.zeros(nu, -(-cap // 64), dtype=torch.int32)
        stack = torch.arange(40 - 1, -1, -1, dtype=torch.int32)
        a = er.pool_alloc(users, jr.packed_counts(ids, off, max_len), L0, pt, stack, 7, nu, cap, 64)
        b = er.pool_alloc(users, (pids != 0).sum(1), L0, pt, stack, 7, nu, cap, 64)
        assert torch.equal(a["page_table"], b["page_table"]) and torch.equal(a["room"], b["room"])
        assert (a["free_top"], a["errors"]) == (b["free_top"], b["errors"])


@pytest.mark.parametrize("seed", range(6))
def test_packed_append_restatement_matches_the_padded_reference(seed):
    g = torch.Generator().manual_seed(seed)
    _check_against_padded(g, 7, 70, idle=seed * 3, pool_users=None, cap=200)
    _check_against_padded(g, 6, 65, idle=5, pool_users=None, cap=200, lengths=[0, 1, 63, 64, 65, 0])
    # a pool: users in any order, one rejected row, rooms that drop items
    _check_against_padded(g, 5, 66, idle=2, pool_users=[4, 0, 7, 2, 3], cap=128,
                          room_rule=lambda b: -1 if b == 3 else [128, 64, 70, 0, 0][b])


def test_clamped_device_offsets():
    """A malformed offsets (past T, decreasing, longer than max_len) is clamped as seq_span clamps it."""
    assert jr.seq_spans([0, 5, 3, 20, 40], 12, 6) == [(0, 5), (5, 0), (3, 6), (12, 0)]
    assert jr.seq_spans([-4, 2], 12, 6) == [(0, 2)]


def test_new_symbols_are_declared_and_bound():
    from genrec_b200 import _lib
    header = open(os.path.join(ROOT, "include", "genrec_b200.h")).read()
    for name in NEW_SYMBOLS:
        assert re.search(r"\b" + name + r"\(", header), name
        assert name in _lib.SIGNATURES, name
