"""Host-side checks of the cached incremental HSTU inference (no GPU): the workspace query of grb_hstu_layer_extend and its
refusals, and, on the fp64 oracle, the two properties the K | V cache relies on."""
import ctypes

import pytest
import torch

from tests.sign_fixed_buckets import use_sign_fixed_oracle


@pytest.fixture(scope="module")
def lib():
    from genrec_b200 import build
    build.build()
    from genrec_b200 import _lib
    return _lib.load()


def test_extend_workspace_bytes_and_errors(lib):
    from genrec_b200._lib import HstuDims
    B, n, D, cap = 128, 1, 128, 256
    d = HstuDims(B, n, D, 4, 32, 64, 0.0, 0, None, 0)
    T = B * n
    ws = lib.grb_hstu_layer_extend_workspace_bytes(ctypes.byref(d), cap)
    # the chunk's activations (as grb_hstu_layer_saved_bytes) + at least one [T, D] fp32 attention partial
    assert ws >= lib.grb_hstu_layer_saved_bytes(ctypes.byref(d)) + T * D * 4
    # a longer cache never needs less scratch
    assert lib.grb_hstu_layer_extend_workspace_bytes(ctypes.byref(d), 4096) >= ws
    for bad, cap_, msg in ((HstuDims(1, 1, 96, 3, 32, 64, 0.0, 0, None, 0), cap, b"unsupported"),
                           (HstuDims(1, 1, 128, 8, 32, 64, 0.0, 0, None, 0), cap, b"head_dim"),
                           (HstuDims(1, 1, 128, 4, 65, 64, 0.0, 0, None, 0), cap, b"num_position_buckets"),
                           (HstuDims(1, 1, 128, 4, 32, 64, 0.1, 0, None, 0), cap, b"dropout_p"),
                           (HstuDims(1, 1, 128, 4, 32, 64, 0.0, 0, None, 0), 0, b"capacity"),
                           (HstuDims(1, 1, 128, 4, 32, 64, 0.0, 0, None, 0), 16385, b"capacity")):
        assert lib.grb_hstu_layer_extend_workspace_bytes(ctypes.byref(bad), cap_) == 0
        assert msg in lib.grb_last_error(), lib.grb_last_error()
    # the entry point itself refuses before touching any pointer
    from genrec_b200._lib import HstuCache, HstuLayerParams
    bad = HstuDims(1, 1, 96, 3, 32, 64, 0.0, 0, None, 0)
    cache = HstuCache(1, cap, 1, None, None, None, None)
    rc = lib.grb_hstu_layer_extend(ctypes.byref(bad), ctypes.byref(HstuLayerParams()), ctypes.byref(cache), 0, None, None, 0, None, None,
                                   None, None, None)
    assert rc == -1 and b"unsupported" in lib.grb_last_error()
    rc = lib.grb_hstu_cache_append(ctypes.byref(HstuCache(1, 0, 1, None, None, None, None)), None, None, 1, None, None, None)
    assert rc == -1


# ---------------------------------------------------------------------------------------------------------------- fp64 oracle
D, H, NB, V = 64, 2, 2, 300


def _params(seed):
    from genrec_b200.hstu import HSTU
    torch.manual_seed(seed)
    m = HSTU(V, 64, D, H, NB, dropout=0.0)
    sd = {k: v.detach().double().clone() for k, v in m.state_dict().items()}
    g = torch.Generator().manual_seed(seed + 1)
    for k in sd:
        if "attention_bias" in k:
            sd[k] = torch.randn(sd[k].shape, generator=g, dtype=torch.float64) * 0.3
    return sd


def _block_outputs(sd, ids, ts):
    import torch.nn.functional as F
    from oracle import hstu as oh
    pad = ids == 0
    x = F.embedding(ids, sd["item_embedding.weight"], padding_idx=0)
    outs = []
    for i in range(NB):
        x = oh.hstu_layer_forward(x, pad, ts, sd, f"layers.{i}.", H)
        outs.append(x)
    return outs


def _history(L, seed):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, V + 1, (2, L), generator=g)
    ts = 1_300_000_000 + torch.cumsum(torch.randint(1, 3 * 86400, (2, L), generator=g), 1)
    ts[:, ::4] = ts[:, ::4] - torch.randint(0, 2, (2, (L + 3) // 4), generator=g)   # some equal / close timestamps
    return ids, ts


@pytest.mark.parametrize("buckets", ["reference", "sign_fixed"])
def test_oracle_appending_items_leaves_earlier_rows_unchanged(buckets, monkeypatch):
    if buckets == "sign_fixed":
        use_sign_fixed_oracle(monkeypatch)
    sd = _params(3)
    ids, ts = _history(40, 4)
    full = _block_outputs(sd, ids, ts)
    for k in (1, 17, 39):
        prefix = _block_outputs(sd, ids[:, :k], ts[:, :k])
        for a, b in zip(prefix, full):
            torch.testing.assert_close(a, b[:, :k], rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("buckets", ["reference", "sign_fixed"])
def test_oracle_valid_rows_do_not_depend_on_left_padding(buckets, monkeypatch):
    if buckets == "sign_fixed":
        use_sign_fixed_oracle(monkeypatch)
    sd = _params(5)
    ids, ts = _history(30, 6)
    base = _block_outputs(sd, ids, ts)
    for m in (1, 9, 64):
        pids = torch.cat([torch.zeros(2, m, dtype=ids.dtype), ids], 1)
        pts = torch.cat([torch.zeros(2, m, dtype=ts.dtype), ts], 1)
        padded = _block_outputs(sd, pids, pts)
        for a, b in zip(padded, base):
            torch.testing.assert_close(a[:, m:], b, rtol=1e-12, atol=1e-12)


def test_sign_fixed_oracle_bias_is_non_uniform(monkeypatch):
    from oracle import hstu as oh
    table = torch.arange(32 * 2, dtype=torch.float64).reshape(32, 2)
    ref = oh.position_bias(table, 40)
    use_sign_fixed_oracle(monkeypatch)
    fixed = oh.position_bias(table, 40)
    causal = torch.tril(torch.ones(40, 40, dtype=torch.bool))
    assert (ref[0][causal] == table[0, 0]).all()                 # the reference: bucket 0 on the whole causal triangle
    assert fixed[0][causal].unique().numel() > 16                 # the sign-fixed table: exact buckets 0..15, then log buckets
    assert fixed[0, 5, 2] == table[3, 0]                          # cell (i, j) -> bucket(i - j)
