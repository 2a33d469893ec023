"""TIGER on packed (jagged) encoder memories: the packed T5 attention core (grb_t5_attention_forward_jagged / _backward_jagged)
against the fp64 reference of tests/attention_reference.py run per sequence, at the query / key tile edges, with idle rows and
dropout; and Tiger.forward_jagged / generate_jagged / retrieve_jagged against the padded entry points on the same users.
`pytest -s` prints each core case's worst and Frobenius ratios (error over the per-element allowance)."""
import math

import numpy as np
import pytest
import torch

from tests import attention_reference as ar
from tests.tiger_params import _geometric_lengths, _model, _padded_and_packed

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
EDGE_LENGTHS = [1, 31, 32, 33, 61, 64, 65, 129]


def _keep(rows, n, p, seed, site):
    """keep-scale matrix [1, H, Lq, n] of the packed kernel's dropout keys `rows` [H, Lq] (uint32), columns 0 .. n - 1"""
    H, Lq = rows.shape
    drop = ar.drop_mask(rows.reshape(-1).astype(np.uint32), n, p, seed, site)
    _, s = ar.keep_scale(p)
    return torch.from_numpy(np.where(drop, 0.0, s)).view(1, H, Lq, n).to(DEV)


def _packed_inputs(lengths, lead, tail, H, dh, Lq, seed):
    g = torch.Generator().manual_seed(seed)
    D = H * dh
    offs = [lead]
    for n in lengths:
        offs.append(offs[-1] + n)
    T = offs[-1] + tail
    B = len(lengths)
    qrows = T if Lq == 0 else B * Lq
    Q = (2 * torch.randn(qrows, D, generator=g)).bfloat16()
    KV = torch.randn(T, 2 * D, generator=g).bfloat16().to(DEV)
    dO = torch.randn(qrows, D, generator=g).bfloat16()
    if Lq:
        Q, dO = Q.view(B, Lq, D), dO.view(B, Lq, D)
    return offs, T, Q.to(DEV), KV[:, :D], KV[:, D:], dO.to(DEV)


def _core_check(tag, lengths, Lq, H, dh, p, lead=0, tail=0, seed=5, site=3):
    """Lq = 0: packed self-attention with a bias table (the encoder); Lq > 0: cross-attention of dense [B, Lq] queries (the decoder)"""
    from genrec_b200 import t5_attention as t5
    offs, T, Q, K, V, dO = _packed_inputs(lengths, lead, tail, H, dh, Lq, sum(lengths) * 7 + Lq + dh)
    max_len = max(lengths)
    scale = 1 / math.sqrt(dh)
    bias = bucket = None
    if Lq == 0:
        bias = (1.5 * torch.randn(H, 32, generator=torch.Generator().manual_seed(3))).to(DEV)
        bucket = t5.relative_position_buckets(max_len, max_len).to(DEV)
    offsets = torch.tensor(offs, dtype=torch.int64, device=DEV)
    out, lse = t5.attention_core_fwd_jagged(Q, K, V, H, bias, bucket, offsets, max_len, False, scale, p, seed, site)
    dq, dk, dv, dbias = t5.attention_core_bwd_jagged(Q, K, V, H, bias, bucket, offsets, max_len, False, scale, out, lse, dO, p, seed, site)
    torch.cuda.synchronize()
    names = ("out", "dq", "dk", "dv")
    got = {n: [] for n in names}
    ref = {k: [] for n in names for k in (n, "a_" + n)}
    db = adb = None
    for b, n in enumerate(lengths):
        r0 = offs[b]
        h = np.arange(H, dtype=np.int64)[:, None]
        if Lq == 0:
            sl = slice(r0, r0 + n)
            q, o, do_ = Q[sl][None], out[sl][None], dO[sl][None]
            rows = (r0 + np.arange(n)[None, :]) * H + h                # token row keys
            bk = t5.relative_position_buckets(n, n).to(DEV)
        else:
            q, o, do_ = Q[b:b + 1], out[b:b + 1], dO[b:b + 1]
            rows = (b * H + h) * Lq + np.arange(Lq)[None, :]            # the padded keys
            bk = None
        keep = _keep(rows, n, p, seed, site)
        saved = ar.attn_keep
        ar.attn_keep = lambda *a, **k: keep
        try:
            r = ar.t5_reference(q, K[r0:r0 + n][None], V[r0:r0 + n][None], H, bias, bk, None, False, scale, do_, o, p, seed, site)
        finally:
            ar.attn_keep = saved
        if Lq == 0:
            got["out"].append(out[r0:r0 + n]); got["dq"].append(dq[r0:r0 + n])
        else:
            got["out"].append(out[b]); got["dq"].append(dq[b])
        got["dk"].append(dk[r0:r0 + n]); got["dv"].append(dv[r0:r0 + n])
        for nm in names:
            ref[nm].append(r[nm][0]); ref["a_" + nm].append(r["a_" + nm][0])
        if bias is not None:
            db = r["dbias"] if db is None else db + r["dbias"]
            adb = r["a_dbias"] if adb is None else adb + r["a_dbias"]
    got = {k: torch.cat(v) for k, v in got.items()}
    ref = {k: torch.cat(v) for k, v in ref.items()}
    if bias is not None:
        got["dbias"], ref["dbias"], ref["a_dbias"] = dbias, db, adb
    err = ar.errors(got, ref, names + ("dbias",))
    print(f"{tag}: {ar.fmt(err)}")
    assert not ar.violations(err, "t5"), ar.fmt(err)
    # idle rows: zeros in out / dq (self-attention) and in dk / dv
    idle = torch.ones(T, dtype=torch.bool, device=DEV)
    idle[offs[0]:offs[-1]] = False
    for t in ((out, dq, dk, dv) if Lq == 0 else (dk, dv)):
        assert not bool(t[idle].any())
    return out, dq, dk, dv, dbias


CORE_CASES = [(Lq, H, dh, p) for Lq, H, dh in ((0, 2, 64), (0, 3, 32), (4, 2, 64), (40, 2, 32)) for p in (0.0, 0.2)]


@pytest.mark.parametrize("Lq,H,dh,p", CORE_CASES)
def test_packed_core_vs_fp64(Lq, H, dh, p):
    _core_check(f"packed t5 Lq={Lq} H={H} dh={dh} p={p}", EDGE_LENGTHS, Lq, H, dh, p)


@pytest.mark.parametrize("Lq", [0, 4])
def test_packed_core_idle_rows(Lq):
    """leading idle rows [0, offsets[0]) and trailing ones past offsets[B], at a single tile and past two"""
    _core_check(f"packed t5 idle Lq={Lq}", [1, 61, 33], Lq, 2, 64, 0.2, lead=3, tail=7)
    _core_check(f"packed t5 idle Lq={Lq} long", [129, 5], Lq, 2, 32, 0.0, lead=1, tail=40)


@pytest.mark.parametrize("Lq,lengths", [(0, [61, 25, 1, 13] * 64), (0, EDGE_LENGTHS * 4), (40, [61, 25, 1, 13] * 64)])
def test_packed_backward_is_reproducible(Lq, lengths):
    from genrec_b200 import t5_attention as t5
    H, dh = 6, 64
    offs, T, Q, K, V, dO = _packed_inputs(lengths, 0, 0, H, dh, Lq, 9)
    max_len = max(lengths)
    bias = bucket = None
    if Lq == 0:
        bias = torch.randn(H, 32, generator=torch.Generator().manual_seed(4)).to(DEV)
        bucket = t5.relative_position_buckets(max_len, max_len).to(DEV)
    offsets = torch.tensor(offs, dtype=torch.int64, device=DEV)
    scale = 1 / math.sqrt(dh)
    out, lse = t5.attention_core_fwd_jagged(Q, K, V, H, bias, bucket, offsets, max_len, False, scale, 0.1, 3, 9)
    a = t5.attention_core_bwd_jagged(Q, K, V, H, bias, bucket, offsets, max_len, False, scale, out, lse, dO, 0.1, 3, 9)
    b = t5.attention_core_bwd_jagged(Q, K, V, H, bias, bucket, offsets, max_len, False, scale, out, lse, dO, 0.1, 3, 9)
    for x, y in zip(a, b):
        if x is not None:
            assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------ models: packed against padded


SHAPES = {"small": ("SMALL", 5, 6), "published": ("PUBLISHED", 256, 20)}


@pytest.mark.parametrize("shape", ["small", "published"])
def test_forward_jagged_equals_forward(shape):
    """dropout 0: logits and loss bit for bit (every row-wise stage sees the same row, and pad keys add exact zeros); the parameter
    gradients to 2e-3 relative Frobenius (the weight-gradient GEMMs sum over the token rows, T of them here and B x width there)"""
    from tests import tiger_params as tp
    name, B, n = SHAPES[shape]
    cfg = dict(getattr(tp, name))
    lengths = None if shape == "small" else _geometric_lengths(B, 1)
    padded, pk = _padded_and_packed(cfg, B, n, 3, lengths)
    m = _model(cfg).train()
    ref = m(padded["user_input_ids"], padded["item_input_ids"], padded["token_type_ids"], padded["target_input_ids"],
            padded["target_token_type_ids"], padded["seq_mask"])
    ref.loss.backward()
    gref = {k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None}
    m.zero_grad(set_to_none=True)
    got = m.forward_jagged(pk["user_input_ids"], pk["item_input_ids"], pk["token_type_ids"], pk["mem_offsets"], pk["max_len"],
                           pk["target_input_ids"], pk["target_token_type_ids"])
    got.loss.backward()
    assert got.logits.shape == ref.logits.shape
    assert torch.equal(got.logits, ref.logits)
    assert torch.equal(got.loss, ref.loss)
    worst = 0.0
    for k, p in m.named_parameters():
        if k not in gref:
            assert p.grad is None or not bool(p.grad.any()), k
            continue
        e = ((p.grad - gref[k]).norm() / gref[k].norm().clamp_min(1e-30)).item()
        worst = max(worst, e)
        assert e < 2e-3, (k, e)
    print(f"{shape}: worst gradient rel. Frobenius error {worst:.2e}")


def test_forward_jagged_backward_is_reproducible():
    from tests import tiger_params as tp
    cfg = dict(tp.PUBLISHED)
    _, pk = _padded_and_packed(cfg, 64, 20, 4, _geometric_lengths(64, 2))
    m = _model(cfg).train()
    grads = []
    for _ in range(2):
        m.zero_grad(set_to_none=True)
        out = m.forward_jagged(pk["user_input_ids"], pk["item_input_ids"], pk["token_type_ids"], pk["mem_offsets"], pk["max_len"],
                               pk["target_input_ids"], pk["target_token_type_ids"])
        out.loss.backward()
        grads.append({k: p.grad.clone() for k, p in m.named_parameters() if p.grad is not None})
    for k in grads[0]:
        assert torch.equal(grads[0][k], grads[1][k]), k


def _gen_setup(shape):
    from tests import tiger_params as tp
    name, B, n = SHAPES[shape]
    cfg = dict(getattr(tp, name))
    B = min(B, 32)
    padded, pk = _padded_and_packed(cfg, B, n, 5, _geometric_lengths(B, 3, cap=n, mean=min(9.0, n / 2)))
    m = _model(cfg).eval()
    valid = torch.randint(0, cfg["num_item_embeddings"], (2000, 3), generator=torch.Generator().manual_seed(2))
    return m, padded, pk, valid


@pytest.mark.parametrize("shape", ["small", "published"])
@pytest.mark.parametrize("K,use_trie", [(10, True), (10, False), (256, True), (256, False)])
def test_generate_jagged_equals_generate(shape, K, use_trie):
    m, padded, pk, valid = _gen_setup(shape)
    gen = torch.Generator(device=DEV)
    gen.manual_seed(K)
    ref = m.generate(padded["user_input_ids"], padded["item_input_ids"], padded["token_type_ids"], padded["seq_mask"],
                     n_top_k_candidates=K, valid_item_ids=valid, use_trie=use_trie, generator=gen)
    gen.manual_seed(K)
    got = m.generate_jagged(pk["user_input_ids"], pk["item_input_ids"], pk["token_type_ids"], pk["mem_offsets"], pk["max_len"],
                            n_top_k_candidates=K, valid_item_ids=valid, use_trie=use_trie, generator=gen)
    assert torch.equal(got.sem_ids, ref.sem_ids)
    assert torch.equal(got.log_probas, ref.log_probas)


def test_retrieve_jagged_equals_retrieve():
    m, padded, pk, valid = _gen_setup("small")
    gen = torch.Generator(device=DEV)
    gen.manual_seed(1)
    ref = m.retrieve(padded["user_input_ids"], padded["item_input_ids"], padded["token_type_ids"], padded["seq_mask"],
                     num_candidates=64, valid_item_ids=valid, generator=gen)
    gen.manual_seed(1)
    got = m.retrieve_jagged(pk["user_input_ids"], pk["item_input_ids"], pk["token_type_ids"], pk["mem_offsets"], pk["max_len"],
                            num_candidates=64, valid_item_ids=valid, generator=gen)
    for x, y in zip(got, ref):
        assert torch.equal(x, y)


def test_generate_jagged_replays_from_a_cuda_graph():
    """a captured generate_jagged at fixed (B, T, max_len) replays with rewritten ids and offsets"""
    from genrec_b200.data import pack_tiger
    from tests import tiger_params as tp
    cfg = dict(tp.SMALL)
    m = _model(cfg).eval()
    valid = torch.randint(0, cfg["num_item_embeddings"], (900, 3), generator=torch.Generator().manual_seed(2))
    B, T = 6, 64

    def packed(seed):
        g = torch.Generator().manual_seed(seed)
        lens = torch.randint(0, 7, (B,), generator=g) * 3
        off = torch.zeros(B + 1, dtype=torch.int64)
        off[1:] = lens.cumsum(0)
        toks = torch.randint(0, cfg["num_item_embeddings"], (int(off[-1]),), generator=g)
        users = torch.randint(0, 500, (B,), generator=g)
        return pack_tiger(users.to(DEV), toks.to(DEV), off.to(DEV), torch.zeros(B, 3, dtype=torch.int64, device=DEV), max_items=6,
                          num_tokens=T)

    first, second = packed(1), packed(2)
    static = {k: first[k].clone() for k in ("user_input_ids", "item_input_ids", "token_type_ids", "mem_offsets")}
    args = lambda: (static["user_input_ids"], static["item_input_ids"], static["token_type_ids"], static["mem_offsets"], first["max_len"])
    m.generate_jagged(*args(), n_top_k_candidates=10, valid_item_ids=valid)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.generate_jagged(*args(), n_top_k_candidates=10)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = m.generate_jagged(*args(), n_top_k_candidates=10)
    for k in static:
        static[k].copy_(second[k])
    state = torch.cuda.get_rng_state()
    graph.replay()
    torch.cuda.synchronize()
    got = (cap.sem_ids.clone(), cap.log_probas.clone())
    torch.cuda.set_rng_state(state)
    eager = m.generate_jagged(second["user_input_ids"], second["item_input_ids"], second["token_type_ids"], second["mem_offsets"],
                              second["max_len"], n_top_k_candidates=10)
    assert not bool(second["overflow"])
    assert torch.equal(got[0], eager.sem_ids) and torch.equal(got[1], eager.log_probas)
