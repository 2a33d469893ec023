"""Packed (jagged) TIGER batches without a GPU: data.pack_tiger against the reference's pad_collate (restated below) with its pads
removed, the argument refusals of Tiger.forward_jagged / generate_jagged / retrieve_jagged, and the new entry points in the header
and the ctypes binding."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def pad_collate(batch, pad_id=0):
    """genrec/trainers/tiger_trainer.py:27-80 (padding_side "left": the items first, the pads behind), restated for dict samples
    {user_id, item_ids (tokens), target_ids}."""
    max_item_length = max(len(x["item_ids"]) for x in batch)
    B = len(batch)
    user_ids = torch.full((B, 1), pad_id, dtype=torch.long)
    ids = torch.full((B, max_item_length), pad_id, dtype=torch.long)
    mask = torch.zeros((B, max_item_length), dtype=torch.long)
    token_type_ids = torch.zeros((B, max_item_length), dtype=torch.long)
    target_input_ids = torch.full((B, len(batch[0]["target_ids"])), pad_id, dtype=torch.long)
    target_token_type_ids = torch.zeros((B, len(batch[0]["target_ids"])), dtype=torch.long)
    for i in range(B):
        item_ids = batch[i]["item_ids"]
        user_ids[i, 0] = batch[i]["user_id"]
        ids[i, :len(item_ids)] = torch.tensor(item_ids, dtype=torch.long)
        token_type_ids[i, :len(item_ids)] = torch.arange(len(item_ids)) % 3
        mask[i, :len(item_ids)] = 1
        target_input_ids[i, :] = torch.tensor(batch[i]["target_ids"])
        target_token_type_ids[i, :] = torch.arange(len(batch[i]["target_ids"]))
    return {"user_input_ids": user_ids, "item_input_ids": ids, "token_type_ids": token_type_ids, "target_input_ids": target_input_ids,
            "target_token_type_ids": target_token_type_ids, "seq_mask": mask}


def _samples(n_items, seed):
    g = torch.Generator().manual_seed(seed)
    return [{"user_id": int(torch.randint(0, 10 ** 5, (1,), generator=g)),
             "item_ids": torch.randint(0, 256, (3 * n,), generator=g).tolist(),
             "target_ids": torch.randint(0, 256, (3,), generator=g).tolist()} for n in n_items]


def _pack(samples, **kw):
    from genrec_b200.data import pack_tiger
    toks = torch.tensor([t for s in samples for t in s["item_ids"]], dtype=torch.int64)
    off = torch.zeros(len(samples) + 1, dtype=torch.int64)
    off[1:] = torch.tensor([len(s["item_ids"]) for s in samples]).cumsum(0)
    return pack_tiger(torch.tensor([s["user_id"] for s in samples], dtype=torch.int64), toks, off,
                      torch.tensor([s["target_ids"] for s in samples], dtype=torch.int64), **kw)


@pytest.mark.parametrize("n_items", [[0], [1], [20], [0, 1, 20, 7, 3], [5, 0, 0, 20, 20, 1]])
def test_pack_tiger_is_pad_collate_without_pads(n_items):
    samples = _samples(n_items, len(n_items))
    ref = pad_collate(samples)
    pk = _pack(samples)
    off = pk["mem_offsets"].tolist()
    assert pk["max_len"] == 1 + 3 * max(n_items) and off[-1] == pk["item_input_ids"].numel() and not bool(pk["overflow"])
    assert torch.equal(pk["user_input_ids"], ref["user_input_ids"].view(-1))
    assert torch.equal(pk["target_input_ids"], ref["target_input_ids"])
    assert torch.equal(pk["target_token_type_ids"], ref["target_token_type_ids"])
    for b, n in enumerate(n_items):
        assert off[b + 1] - off[b] == 1 + 3 * n                                          # the user row, then the items
        keep = ref["seq_mask"][b].bool()
        assert torch.equal(pk["item_input_ids"][off[b] + 1:off[b + 1]], ref["item_input_ids"][b][keep])
        assert torch.equal(pk["token_type_ids"][off[b] + 1:off[b + 1]], ref["token_type_ids"][b][keep])
        assert int(pk["item_input_ids"][off[b]]) == 0 and int(pk["token_type_ids"][off[b]]) == 0


def test_pack_tiger_keeps_the_last_max_items():
    samples = _samples([25, 4], 3)
    pk = _pack(samples, max_items=20)
    off = pk["mem_offsets"].tolist()
    assert off == [0, 61, 74] and pk["max_len"] == 61
    assert pk["item_input_ids"][1:61].tolist() == samples[0]["item_ids"][-60:]
    assert pk["token_type_ids"][1:61].tolist() == [i % 3 for i in range(60)]


def test_pack_tiger_fixed_rows_and_overflow():
    samples = _samples([2, 3], 4)
    pk = _pack(samples, max_items=20, num_tokens=20)
    assert pk["item_input_ids"].numel() == 20 and pk["max_len"] == 61 and not bool(pk["overflow"])
    assert pk["mem_offsets"].tolist() == [0, 7, 17]
    assert not bool(pk["item_input_ids"][17:].any()) and not bool(pk["token_type_ids"][17:].any())   # idle rows
    cut = _pack(samples, max_items=20, num_tokens=10)
    assert bool(cut["overflow"]) and cut["mem_offsets"].tolist() == [0, 7, 10]
    assert torch.equal(cut["item_input_ids"], pk["item_input_ids"][:10])


def test_pack_tiger_refuses_bad_inputs():
    from genrec_b200.data import pack_tiger
    i64 = lambda *a: torch.tensor(a, dtype=torch.int64)
    with pytest.raises(ValueError, match="int64"):
        pack_tiger(i64(1), torch.zeros(3, dtype=torch.int32), i64(0, 3), torch.zeros(1, 3, dtype=torch.int64))
    with pytest.raises(ValueError, match="user_ids"):
        pack_tiger(i64(1, 2), i64(1, 2, 3), i64(0, 3), torch.zeros(1, 3, dtype=torch.int64))
    with pytest.raises(ValueError, match="num_tokens"):
        pack_tiger(i64(1), i64(1, 2, 3), i64(0, 3), torch.zeros(1, 3, dtype=torch.int64), num_tokens=0)


def _tiger():
    from genrec_b200.tiger import Tiger
    from tests import tiger_params as tp
    return Tiger(**tp.SMALL)


def _args(offsets=(0, 4, 8), max_len=4, T=8, users=2, types=None):
    ids = torch.zeros(T, dtype=torch.int64)
    return (torch.arange(users, dtype=torch.int64), ids, ids.clone() if types is None else types, torch.tensor(offsets, dtype=torch.int64),
            max_len)


@pytest.mark.parametrize("call", ["forward", "generate", "retrieve"])
@pytest.mark.parametrize("kw, msg", [
    (dict(offsets=(1, 4, 8)), "offsets\\[0\\] must be 0"),
    (dict(offsets=(0, 5, 4)), "non-decreasing"),
    (dict(offsets=(0, 5, 8)), "exceeds max_len"),
    (dict(offsets=(0, 4, 9), max_len=5), "exceeds the 8 token rows"),
    (dict(offsets=(0, 0, 4)), "user row"),
    (dict(max_len=0), "max_len"),
    (dict(max_len=4096), "max_len"),
    (dict(users=3), "3 user ids for 2 sequences"),
    (dict(types=torch.zeros(7, dtype=torch.int64)), "token_type_ids"),
])
def test_jagged_entry_points_refuse_before_any_launch(call, kw, msg):
    m = _tiger()
    a = _args(**kw)
    with pytest.raises(ValueError, match=msg):
        if call == "forward":
            m.forward_jagged(*a, torch.zeros(2, 3, dtype=torch.int64), torch.zeros(2, 3, dtype=torch.int64))
        elif call == "generate":
            m.generate_jagged(*a)
        else:
            m.retrieve_jagged(*a)


def test_jagged_refuses_more_than_65535_users():
    m = _tiger()
    B = 65536
    off = torch.arange(B + 1, dtype=torch.int64)
    with pytest.raises(ValueError, match="65535"):
        m.generate_jagged(torch.zeros(B, dtype=torch.int64), torch.zeros(B, dtype=torch.int64), torch.zeros(B, dtype=torch.int64), off, 1)


def test_new_symbols_are_declared_and_bound():
    from genrec_b200 import _lib
    header = open(os.path.join(ROOT, "include", "genrec_b200.h")).read()
    for name in ("grb_t5_attention_forward_jagged", "grb_t5_attention_backward_jagged", "grb_t5_attention_backward_workspace_bytes_jagged"):
        assert re.search(r"\b" + name + r"\(", header), name
        assert name in _lib.SIGNATURES, name
        assert hasattr(_lib.load(), name), name                                           # exported by the built library
