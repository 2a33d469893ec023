"""Packed (jagged) HSTU batches without a GPU: the argument refusals of HSTU.forward_jagged / evaluate_batch_jagged, and the fp64
attention reference of tests/hstu_block_reference.py run per sequence on a packed batch against the same reference on the
left-padded batch (HSTU has no absolute position embedding, so the two must agree on every real token)."""
import pytest
import torch

from tests import hstu_block_reference as hr

LENGTHS = [1, 5, 63, 64, 65, 70]


def _model(**kw):
    from genrec_b200.hstu import HSTU
    torch.manual_seed(0)
    return HSTU(50, 80, 64, 2, 1, dropout=0.0, **kw)


def _ids(T):
    return torch.randint(1, 51, (T,), dtype=torch.int64)


@pytest.mark.parametrize("offsets, max_len, T, msg", [
    ([1, 3, 5], 4, 5, "offsets\\[0\\] must be 0"),
    ([0, 3, 2], 4, 5, "non-decreasing"),
    ([0, 3, 9], 4, 9, "exceeds max_len"),
    ([0, 3, 6], 4, 5, "exceeds the 5 token rows"),
])
def test_forward_jagged_refuses_a_malformed_cpu_batch(offsets, max_len, T, msg):
    m = _model()
    off = torch.tensor(offsets, dtype=torch.int64)
    with pytest.raises(ValueError, match=msg):
        m.forward_jagged(_ids(T), off, max_len)
    with pytest.raises(ValueError, match=msg):
        m.evaluate_batch_jagged(_ids(T), off, max_len, None, torch.ones(len(offsets) - 1, dtype=torch.int64))


@pytest.mark.parametrize("bad", ["max_len0", "max_len_big", "ids_2d", "offsets_short", "offsets_i32", "ts_shape", "targets_shape"])
def test_forward_jagged_refuses_bad_shapes(bad):
    m = _model()
    ids, off, max_len, ts, tg = _ids(6), torch.tensor([0, 2, 6]), 4, None, None
    if bad == "max_len0":
        max_len = 0
    elif bad == "max_len_big":
        max_len = 16385
    elif bad == "ids_2d":
        ids = ids.view(2, 3)
    elif bad == "offsets_short":
        off = torch.tensor([0])
    elif bad == "offsets_i32":
        off = off.int()
    elif bad == "ts_shape":
        ts = torch.zeros(5, dtype=torch.int64)
    else:
        tg = torch.zeros(5, dtype=torch.int64)
    with pytest.raises(ValueError):
        m.forward_jagged(ids, off, max_len, ts, tg)


def test_forward_jagged_refuses_more_than_65535_sequences():
    """B = 65,536 sequences of length 1 is a well-formed batch, but the attention grid holds at most 65,535 sequences: the refusal
    comes before the embedding launches."""
    m = _model()
    B = 65536
    off = torch.arange(B + 1, dtype=torch.int64)
    with pytest.raises(ValueError, match="65535"):
        m.forward_jagged(_ids(B), off, 1)
    with pytest.raises(ValueError, match="65535"):
        m.evaluate_batch_jagged(_ids(B), off, 1, None, torch.ones(B, dtype=torch.int64))


def test_jagged_paths_refuse_fp32_precision():
    m = _model().set_precision("fp32")
    off = torch.tensor([0, 2, 6])
    with pytest.raises(RuntimeError, match="bf16"):
        m.forward_jagged(_ids(6), off, 4)
    with pytest.raises(RuntimeError, match="bf16"):
        m.evaluate_batch_jagged(_ids(6), off, 4, None, torch.ones(2, dtype=torch.int64))


def _index(ts, pad, pb, thr, nt, npos):
    """[B, L, L] bias index of grb_hstu_bias_index restated on the host (sentinel npos * 64 for masked cells)."""
    B, L = pad.shape
    i = torch.arange(L)
    d = (ts[:, :, None] - ts[:, None, :]).abs().clamp(min=1)
    tb = torch.bucketize(d, thr[1:64], right=True).clamp(max=nt - 1)
    idx = pb[(i[:, None] - i[None, :]).clamp(min=0)][None] * 64 + tb
    valid = (i[None, :] <= i[:, None])[None] & ~pad[:, None, :]
    return torch.where(valid, idx, torch.full_like(idx, npos * 64)), valid[:, None]


@pytest.mark.parametrize("H", [2, 4])
def test_reference_attention_per_sequence_equals_the_padded_batch(H):
    """The reference's own consistency check: every real token of a packed sequence gets the padded batch's O, dQ, dK, dV and dS."""
    from genrec_b200.hstu import time_bucket_thresholds
    g = torch.Generator().manual_seed(3)
    D, L, B, nt, npos = 64, max(LENGTHS), len(LENGTHS), 20, 16
    thr = time_bucket_thresholds()
    pb = torch.randint(0, npos, (L,), generator=g)
    wpos, wtime = 0.3 * torch.randn(npos, H, generator=g), 0.5 * torch.randn(nt, H, generator=g)
    pad = torch.ones(B, L, dtype=torch.bool)
    for b, n in enumerate(LENGTHS):
        pad[b, L - n:] = False
    ts = torch.where(pad, 0, 1_300_000_000 + torch.cumsum(torch.randint(1, 10 ** 6, (B, L), generator=g), 1))
    P = (0.5 * torch.randn(B, L, 4 * D, generator=g)).bfloat16()
    zp = (0.5 * torch.randn(B, L, 4 * D, generator=g)).bfloat16()
    dO = (0.5 * torch.randn(B, L, D, generator=g)).bfloat16()
    idx, valid = _index(ts, pad, pb, thr, nt, npos)
    w, masked, _, _ = hr.cell_bias(idx, wpos, wtime, npos, H)
    assert torch.equal(masked, ~valid)
    full = hr.attention(P, w, valid, H, zp, dO)
    for b, n in enumerate(LENGTHS):
        s = slice(L - n, L)
        pidx, pvalid = _index(ts[b:b + 1, s], pad[b:b + 1, s], pb, thr, nt, npos)
        pw, _, _, _ = hr.cell_bias(pidx, wpos, wtime, npos, H)
        one = hr.attention(P[b:b + 1, s], pw, pvalid, H, zp[b:b + 1, s], dO[b:b + 1, s])
        for k in ("O", "dQ", "dK", "dV"):
            torch.testing.assert_close(one[k][0], full[k][b, s], rtol=1e-12, atol=1e-12, msg=k)
            # the allowances carry the fp32 summation depth, which is the sequence's own length once the pads are gone
            assert bool((one["a_" + k][0] <= full["a_" + k][b, s] * (1 + 1e-12)).all()), k
        torch.testing.assert_close(one["dS"][0], full["dS"][b, :, s, s], rtol=1e-12, atol=1e-12)
