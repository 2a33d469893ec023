"""Packed (jagged) SASRec batches without a GPU: the argument refusals of SASRec.forward_jagged / evaluate_batch_jagged, the position
rule (item i of a sequence of packed length n sits at position P - n + i, P the batch's longest packed sequence) against the
positions sasrec_collate_fn and the evaluation collate give, and the fp64 SASRec attention reference run per sequence against its
run on the left-padded batch."""
import pytest
import torch

from tests import attention_reference as ar

MAX_SEQ_LEN = 8


def _model():
    from genrec_b200.sasrec import SASRec
    torch.manual_seed(0)
    return SASRec(50, MAX_SEQ_LEN, 64, 2, 1, 128, dropout=0.0)


def _ids(T):
    return torch.randint(1, 51, (T,), dtype=torch.int64)


def packed_positions(lengths, max_seq_len):
    """The position rule restated: each history keeps its last n = min(len, max_seq_len) items; P = max n; item i -> P - n + i."""
    ns = [min(n, max_seq_len) for n in lengths]
    P = max(ns)
    return [[P - n + i for i in range(n)] for n in ns], P


@pytest.mark.parametrize("offsets, max_len, T, msg", [
    ([1, 3, 5], 4, 5, "offsets\\[0\\] must be 0"),
    ([0, 3, 2], 4, 5, "non-decreasing"),
    ([0, 3, 8], 4, 8, "exceeds max_len"),
    ([0, 3, 6], 4, 5, "exceeds the 5 token rows"),
])
def test_forward_jagged_refuses_a_malformed_cpu_batch(offsets, max_len, T, msg):
    m = _model()
    off = torch.tensor(offsets, dtype=torch.int64)
    with pytest.raises(ValueError, match=msg):
        m.forward_jagged(_ids(T), off, max_len)
    with pytest.raises(ValueError, match=msg):
        m.evaluate_batch_jagged(_ids(T), off, max_len, torch.ones(len(offsets) - 1, dtype=torch.int64))


@pytest.mark.parametrize("bad", ["max_len0", "max_len_over_table", "max_len_float", "ids_2d", "ids_i32", "offsets_short", "offsets_i32",
                                 "targets_shape", "eval_targets_shape"])
def test_forward_jagged_refuses_bad_shapes(bad):
    m = _model()
    ids, off, max_len, tg = _ids(6), torch.tensor([0, 2, 6]), 4, None
    eval_tg = torch.ones(2, dtype=torch.int64)
    if bad == "max_len0":
        max_len = 0
    elif bad == "max_len_over_table":
        max_len = MAX_SEQ_LEN + 1            # the position table has max_seq_len rows
    elif bad == "max_len_float":
        max_len = 4.0
    elif bad == "ids_2d":
        ids = ids.view(2, 3)
    elif bad == "ids_i32":
        ids = ids.int()
    elif bad == "offsets_short":
        off = torch.tensor([0])
    elif bad == "offsets_i32":
        off = off.int()
    elif bad == "targets_shape":
        tg = torch.zeros(5, dtype=torch.int64)
    else:
        eval_tg = torch.ones(3, dtype=torch.int64)
    with pytest.raises(ValueError):
        if bad == "eval_targets_shape":
            m.evaluate_batch_jagged(ids, off, max_len, eval_tg)
        else:
            m.forward_jagged(ids, off, max_len, tg)
    if bad not in ("targets_shape", "eval_targets_shape"):
        with pytest.raises(ValueError):
            m.evaluate_batch_jagged(ids, off, max_len, torch.ones(max(off.numel() - 1, 1), dtype=torch.int64))


@pytest.mark.parametrize("where", ["cpu", "device"])
def test_forward_jagged_refuses_more_than_65535_sequences(where):
    """B = 65,536 sequences of length 1 is refused before any launch.  For offsets that live on a device the refusal reads no value:
    a tensor on the 'meta' device, which has no values to read, stands in for device offsets here."""
    m = _model()
    B = 65536
    off = torch.arange(B + 1, dtype=torch.int64)
    if where == "device":
        off = off.to("meta")
    with pytest.raises(ValueError, match="65535"):
        m.forward_jagged(_ids(B), off, 1)
    with pytest.raises(ValueError, match="65535"):
        m.evaluate_batch_jagged(_ids(B), off, 1, torch.ones(B, dtype=torch.int64))


def _histories(lengths, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(1, 1000, (n,), generator=g).tolist() for n in lengths], torch.randint(1, 1000, (len(lengths),), generator=g).tolist()


@pytest.mark.parametrize("lengths", [
    [3, 1, 5, 2],            # longest below max_seq_len
    [8, 3, 8, 1],            # at max_seq_len
    [12, 3, 9, 1, 20],       # above: every history is cut to its last max_seq_len items
    [0, 4, 0, 6],            # empty histories
    [0, 11, 1],
])
def test_position_rule_matches_the_padded_collates(lengths):
    """Every item of the packed batch sits, in sasrec_collate_fn's and in the evaluation collate's left-padded rows, at the position
    the rule gives it: same id, same target, and only pads elsewhere.  The padded batch is P wide."""
    from genrec_b200.data import hstu_eval_collate_fn, sasrec_collate_fn
    hist, tgt = _histories(lengths)
    pos, P = packed_positions(lengths, MAX_SEQ_LEN)
    rows = [dict(history=h, target=t) for h, t in zip(hist, tgt)]
    train = sasrec_collate_fn(rows, MAX_SEQ_LEN)
    ev = hstu_eval_collate_fn([dict(history=h, timestamps=[0] * len(h), target=t) for h, t in zip(hist, tgt)], MAX_SEQ_LEN)
    assert train["input_ids"].shape == (len(lengths), P) and ev["input_ids"].shape == (len(lengths), P)
    assert torch.equal(ev["targets"], torch.tensor(tgt))
    for b, (h, t) in enumerate(zip(hist, tgt)):
        n = len(pos[b])
        items = h[len(h) - n:]
        targets = items[1:] + [t] if n else []
        cols = torch.tensor(pos[b], dtype=torch.long)
        for batch in (train, ev):
            ids = batch["input_ids"][b]
            assert ids[cols].tolist() == items
            others = torch.ones(P, dtype=torch.bool)
            others[cols] = False
            assert bool((ids[others] == 0).all())
        assert train["targets"][b, cols].tolist() == targets
        # the shift gives the last pad row (position P - n - 1) the first item as its target; a packed batch has no such row
        if n < P:
            first = items[0] if n else t
            assert int(train["targets"][b, P - n - 1]) == first


@pytest.mark.parametrize("H, dh", [(2, 32), (1, 64)])
def test_reference_attention_per_sequence_equals_the_padded_batch(H, dh):
    """sasrec_reference (dropout off) on each sequence alone gives the padded batch's O, dQ, dK, dV on its real rows; id-0 tokens
    inside a sequence stay masked keys and zeroed queries."""
    g = torch.Generator().manual_seed(4)
    lengths = [1, 5, 63, 64, 65, 70]
    B, L, D = len(lengths), max(lengths), H * dh
    pad = torch.ones(B, L, dtype=torch.uint8)
    for b, n in enumerate(lengths):
        pad[b, L - n:] = 0
    pad[2, L - 63 + 7] = 1                            # an id 0 inside a sequence
    pad[4, L - 1] = 1
    Q, K, V, dO = [(0.7 * torch.randn(B, L, D, generator=g)).bfloat16() for _ in range(4)]
    full = ar.sasrec_reference(Q, K, V, pad, H)
    O = full["out"].bfloat16()
    full = ar.sasrec_reference(Q, K, V, pad, H, dO, O)
    for b, n in enumerate(lengths):
        s = slice(L - n, L)
        one = ar.sasrec_reference(Q[b:b + 1, s], K[b:b + 1, s], V[b:b + 1, s], pad[b:b + 1, s], H, dO[b:b + 1, s], O[b:b + 1, s])
        for k in ("out", "dq", "dk", "dv"):
            torch.testing.assert_close(one[k][0], full[k][b, s], rtol=1e-12, atol=1e-12, msg=k)
            # the allowances carry the fp32 summation depth, which is the sequence's own length once the pads are gone
            assert bool((one["a_" + k][0] <= full["a_" + k][b, s] * (1 + 1e-12)).all()), k
        torch.testing.assert_close(one["lse"][0], full["lse"][b, :, s], rtol=1e-12, atol=1e-12)
