"""TIGER's wide beam step (csrc/beam.cuh, grb_beam_select_wide) against the oracle restatement of the reference's greedy scan
(oracle/tiger_decode.select), bit for bit: sequences, totals and trie nodes.  Then end to end through Tiger.generate / retrieve at
retrieval widths, and the T5 attention forward past 65,535 (batch, head) pairs."""
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _walk(csr, seq):
    off, tok, child = csr
    nd = 0
    for t in seq:
        nxt = -1
        for e in range(off[nd], off[nd + 1]):
            if tok[e] == t:
                nxt = child[e]
                break
        if nxt < 0:
            return -1
        nd = nxt
    return nd


def _csr_ids(root, trie):
    """id(dict node of the oracle's trie) -> CSR node id, by walking both tries together."""
    from oracle import tiger_decode as od
    off, tok, child = trie.child_off.tolist(), trie.child_tok.tolist(), trie.child_node.tolist()
    ids, stack = {id(root): 0, id(od.DEAD_NODE): -1}, [(root, 0)]
    while stack:
        nd, c = stack.pop()
        for e in range(off[c], off[c + 1]):
            ids[id(nd[tok[e]])] = child[e]
            stack.append((nd[tok[e]], child[e]))
    return ids


def _case(K, num_emb, S, use_trie, seed, leaf=False):
    """Three batch rows.  Row 0: a wide set of parents with identical parents inside it, a dead parent, repeated and out-of-range
    tokens (negative ones included) in some parents, -inf and -5e32 totals and exact ties.  Row 1: every parent identical.  Row 2:
    every parent identical and only five distinct tokens: fewer distinct candidates than K."""
    from oracle import tiger_decode as od
    from genrec_b200 import tiger_decode as td
    g = torch.Generator().manual_seed(seed)
    KK = min(6 * K, num_emb)
    B = 3
    depth = S if leaf else 3                   # leaf: every parent on the trie is a leaf, so every child is dead
    valid = torch.randint(0, num_emb, (4000, depth), generator=g)
    valid[:300, 0] = 7
    seqs = valid[torch.randint(0, 4000, (B, K), generator=g)][:, :, :S].contiguous()
    if S > 0:
        seqs[0, 3::7] = seqs[0, 1]
        seqs[0, 2] = 999
        seqs[1:] = seqs[1:, :1]
    q = lambda *shape: -torch.randint(0, 12, shape, generator=g).float() / 4       # noqa: E731  (exact ties)
    beam_logps = q(B, K)
    beam_logps[0, 5] = float("-inf")
    beam_logps[1:] = beam_logps[1:, :1]
    tok = torch.stack([torch.stack([torch.randperm(num_emb, generator=g)[:KK] for _ in range(K)]) for _ in range(B)])
    tok[0, ::3] = torch.randint(-40, num_emb + 40, (len(range(0, K, 3)), KK), generator=g)
    tok[2] = torch.randint(0, 5, (K, KK), generator=g)
    logp = q(B, K, KK) - torch.rand(B, K, KK, generator=g).mul(4).floor().mul(0.5)
    logp[0, 1::4, ::5] = -5e32
    logp[0, 2::4, 1::5] = float("-inf")
    logp[1, :, -KK // 3:] = -5e32
    root = od.build_trie(valid) if use_trie else None
    trie = td.TrieCSR.build(valid).to(DEV) if use_trie else None
    nodes_o, nodes_g = None, None
    if use_trie:
        nodes_o = [[root] * K for _ in range(B)]
        for b in range(B):
            for k in range(K):
                nd = root
                for t in seqs[b, k].tolist():
                    nd = nd.get(t, od.DEAD_NODE)
                nodes_o[b][k] = nd
        csr = trie.child_off.tolist(), trie.child_tok.tolist(), trie.child_node.tolist()
        nodes_g = torch.tensor([[_walk(csr, seqs[b, k].tolist()) for k in range(K)] for b in range(B)], dtype=torch.int32, device=DEV)
    return seqs, beam_logps, tok, logp, root, nodes_o, trie, nodes_g


def _check(K, num_emb, S, use_trie, seed, leaf=False):
    from oracle import tiger_decode as od
    from genrec_b200 import tiger_decode as td
    seqs, beam_logps, tok, logp, root, nodes_o, trie, nodes_g = _case(K, num_emb, S, use_trie, seed, leaf)
    so, lo, no = od.select(seqs, beam_logps, tok, logp, nodes_o, root, use_trie)
    sg, lg, ng = td.beam_select(seqs.to(DEV), beam_logps.to(DEV), tok.to(DEV), logp.to(DEV), nodes_g, trie)
    assert torch.equal(sg.cpu(), so)
    assert torch.equal(lg.cpu(), lo)
    if use_trie:
        ids = _csr_ids(root, trie)
        want = torch.tensor([[ids[id(n)] for n in row] for row in no], dtype=torch.int32)
        assert torch.equal(ng.cpu(), want)
        if leaf:
            assert (want == -1).any()                  # children of leaves
    else:
        assert ng is None
    return so, lo


WIDTHS = [(14, 256), (64, 256), (256, 256), (1024, 256), (14, 1024), (64, 1024), (256, 1024)]   # K * min(6 K, num_emb) <= 262,144


@pytest.mark.parametrize("K, num_emb", WIDTHS)
@pytest.mark.parametrize("S", [0, 1, 2])
@pytest.mark.parametrize("use_trie", [True, False])
def test_wide_beam_select_vs_oracle(K, num_emb, S, use_trie):
    so, lo = _check(K, num_emb, S, use_trie, seed=K + num_emb + 10 * S + use_trie)
    assert (lo[2] == -1e32).any()                      # row 2 ran out of distinct candidates: fillers


@pytest.mark.parametrize("S", [1, 2])
def test_wide_beam_select_from_leaf_nodes(S):
    _check(64, 256, S, True, seed=S, leaf=True)


# ---- end to end
def _small(K_seed=0):
    from genrec_b200.tiger import Tiger
    from tests import tiger_params as tp
    cfg = dict(tp.SMALL)
    m = Tiger(**cfg)
    m.load_state_dict(tp.tiger_params([(k, v.shape) for k, v in m.state_dict().items()], 7))
    m = m.to(DEV).eval()
    b = {k: v.to(DEV) for k, v in tp.batch(cfg, 3, 6, 11 + K_seed).items()}
    valid = torch.randint(0, cfg["num_item_embeddings"], (900, 3), generator=torch.Generator().manual_seed(2))
    return m, (b["user_input_ids"], b["item_input_ids"], b["token_type_ids"], b["seq_mask"]), valid


@pytest.mark.parametrize("K", [20, 64, 256])
def test_generate_replays_as_the_oracle_loop(K, monkeypatch):
    """Tiger.generate with its logits and torch.multinomial draws recorded, then the oracle's loop on the same logits and draws."""
    from oracle import tiger_decode as od
    from genrec_b200 import tiger_decode as td
    m, args, valid = _small(K)
    logits, draws = [], []
    sm, mn = td.trie_log_softmax, torch.multinomial
    monkeypatch.setattr(td, "trie_log_softmax", lambda x, *a: (logits.append(x.cpu()), sm(x, *a))[1])
    monkeypatch.setattr(torch, "multinomial", lambda *a, **k: (lambda r: (draws.append(r.cpu()), r)[1])(mn(*a, **k)))
    gen = torch.Generator(device=DEV).manual_seed(K)
    out = m.generate(*args, n_top_k_candidates=K, valid_item_ids=valid, generator=gen)
    monkeypatch.undo()
    seqs, logps = od.replay(logits, draws, valid, 3, K, m.num_item_embeddings, 0.2)
    assert torch.equal(out.sem_ids.cpu(), seqs)
    torch.testing.assert_close(out.log_probas.cpu(), logps, rtol=1e-5, atol=1e-5)


def test_generate_equals_the_uncached_loop_at_width_64():
    from genrec_b200 import tiger_decode as td
    m, args, valid = _small()
    gen = torch.Generator(device=DEV)
    gen.manual_seed(5)
    ours = m.generate(*args, n_top_k_candidates=64, valid_item_ids=valid, generator=gen)
    gen.manual_seed(5)
    ref = td.generate(m, *args, n_top_k_candidates=64, generator=gen)
    assert torch.equal(ours.sem_ids, ref.sem_ids) and torch.equal(ours.log_probas, ref.log_probas)


def test_generate_at_width_256_in_a_cuda_graph():
    m, args, valid = _small()
    m.generate(*args, n_top_k_candidates=256, valid_item_ids=valid)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m.generate(*args, n_top_k_candidates=256)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        cap = m.generate(*args, n_top_k_candidates=256)
    state = torch.cuda.get_rng_state()
    graph.replay()
    torch.cuda.synchronize()
    got = (cap.sem_ids.clone(), cap.log_probas.clone())
    torch.cuda.set_rng_state(state)
    eager = m.generate(*args, n_top_k_candidates=256)
    assert torch.equal(got[0], eager.sem_ids) and torch.equal(got[1], eager.log_probas)


@pytest.mark.parametrize("K", [10, 300])
def test_retrieve_rows_are_the_leaf_lookup(K):
    m, args, valid = _small()
    valid[500:520] = valid[3]                            # a duplicated tuple: its smallest row is 3
    gen = torch.Generator(device=DEV)
    gen.manual_seed(9)
    items, sem_ids, logps = m.retrieve(*args, num_candidates=K, valid_item_ids=valid, generator=gen)
    gen.manual_seed(9)
    out = m.generate(*args, n_top_k_candidates=K, generator=gen)
    assert torch.equal(sem_ids, out.sem_ids) and torch.equal(logps, out.log_probas)
    first = {}
    for i, r in enumerate(valid.tolist()):
        first.setdefault(tuple(r), i)
    want = torch.tensor([[first.get(tuple(s), -1) if lp > -1e32 else -1 for s, lp in zip(sb.tolist(), lb.tolist())]
                         for sb, lb in zip(sem_ids.cpu(), logps.cpu())])
    assert items.dtype == torch.int64 and torch.equal(items.cpu(), want)
    assert (items >= 0).any()


def test_t5_attention_forward_past_65535_batch_heads():
    """B * H = 66,000 in one launch against the same rows run as chunks that launched before: the same bits."""
    from genrec_b200.t5_attention import _bucket_map, attention_core_fwd
    g = torch.Generator().manual_seed(3)
    B, H, L, DH, nb = 11000, 6, 4, 64, 32
    D = H * DH
    q, k, v = [(torch.randn(B, L, D, generator=g) * 0.5).bfloat16().to(DEV) for _ in range(3)]
    bias = torch.randn(H, nb, generator=g).to(DEV)
    bucket = _bucket_map(L, L, nb, 128, DEV)
    whole, lse = attention_core_fwd(q, k, v, H, bias, bucket, None, True, DH ** -0.5)
    parts = [attention_core_fwd(q[i:i + 5000], k[i:i + 5000], v[i:i + 5000], H, bias, bucket, None, True, DH ** -0.5)
             for i in range(0, B, 5000)]
    assert torch.equal(whole, torch.cat([p[0] for p in parts]))
    assert torch.equal(lse, torch.cat([p[1] for p in parts]))
