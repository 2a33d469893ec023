"""TIGER's wide beam step without a GPU: the width limits are refused before anything runs (Python and C ABI), and the trie's leaf
rows are the smallest catalog rows holding each tuple."""
import ctypes

import pytest
import torch

from genrec_b200 import tiger_decode as td
from tests import tiger_params as tp


@pytest.mark.parametrize("K, num_emb, limit", [(0, 256, "1 .. 1024"), (1025, 256, "1 .. 1024"), (300, 1024, "262144")])
def test_refused_before_the_encoder_runs(K, num_emb, limit):
    """The model and the batch stay on the CPU: any launch, or the encoder, would fail with something other than ValueError."""
    from genrec_b200.tiger import Tiger
    m = Tiger(**dict(tp.SMALL, num_item_embeddings=num_emb))
    b = tp.batch(tp.SMALL, 2, 4, 0)
    args = (b["user_input_ids"], b["item_input_ids"], b["token_type_ids"], b["seq_mask"])
    valid = torch.randint(0, num_emb, (50, 3))
    with pytest.raises(ValueError, match=limit):
        m.generate(*args, n_top_k_candidates=K, valid_item_ids=valid)
    with pytest.raises(ValueError, match=limit):
        m.retrieve(*args, num_candidates=K, valid_item_ids=valid)
    with pytest.raises(ValueError, match=limit):
        td.generate(m, *args, n_top_k_candidates=K, valid_item_ids=valid)
    assert not hasattr(m, "_grb_trie")                   # refused before the trie was built, too


@pytest.mark.parametrize("K, KK", [(0, 6), (1025, 1), (1024, 257), (1, 262145)])
def test_beam_select_refuses_the_width(K, KK):
    B, S = 1, 1
    with pytest.raises(ValueError):
        td.beam_select(torch.zeros(B, max(K, 1), S, dtype=torch.long), torch.zeros(B, max(K, 1)), torch.zeros(B, K, KK, dtype=torch.long),
                       torch.zeros(B, K, KK), None, None)


def test_c_abi_refuses_the_width():
    from genrec_b200 import _lib
    lib = _lib.load()
    assert lib.grb_beam_select_wide_workspace_bytes(256, 1024, 256) > 0
    fake = 16                                            # never dereferenced: the shape is refused first
    for K, KK in ((0, 6), (1025, 1), (1024, 257)):
        assert lib.grb_beam_select_wide_workspace_bytes(4, K, KK) == 0
        rc = lib.grb_beam_select_wide(fake, fake, fake, fake, None, None, None, None, 0, 4, K, KK, 1, fake, fake, None, fake, None)
        assert rc != 0
        assert b"K*KK <= 262144" in lib.grb_last_error()


def _brute_rows(valid, tuples):
    rows = valid.tolist()
    return [min((i for i, r in enumerate(rows) if tuple(r) == t), default=-1) for t in tuples]


@pytest.mark.parametrize("depth", [1, 3])
def test_leaf_rows_against_a_search_of_the_catalog(depth):
    g = torch.Generator().manual_seed(depth)
    valid = torch.randint(0, 6, (300, depth), generator=g)
    valid[100:110] = valid[7]                            # duplicate tuples: the smallest row wins
    valid[250] = valid[299]
    trie = td.TrieCSR.build(valid)
    # walk every leaf of the CSR and read the tuple off the path
    off, tok, child = trie.child_off.tolist(), trie.child_tok.tolist(), trie.child_node.tolist()
    leaves, stack = {}, [(0, ())]
    while stack:
        nd, path = stack.pop()
        if len(path) == depth:
            leaves[nd] = path
        for e in range(off[nd], off[nd + 1]):
            stack.append((child[e], path + (tok[e],)))
    assert len(leaves) == len({tuple(r) for r in valid.tolist()})
    nodes = sorted(leaves)
    want = _brute_rows(valid, [leaves[n] for n in nodes])
    assert trie.leaf_row[nodes].tolist() == want
    inner = [n for n in range(trie.n_nodes) if n not in leaves]
    assert (trie.leaf_row[inner] == -1).all()
    assert trie.rows(torch.tensor([-1, 0] + nodes[:3])).tolist() == [-1, -1] + want[:3]


def test_leaf_rows_of_a_three_dimensional_catalog():
    valid = torch.tensor([[[1, 2], [3, 4]], [[1, 2], [0, 0]]])
    trie = td.TrieCSR.build(valid)
    assert sorted(r for r in trie.leaf_row.tolist() if r >= 0) == [0, 1, 3]     # rows of valid.view(-1, 2); [1, 2] first at row 0
