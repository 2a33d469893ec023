"""genrec_b200.cobra's paged pool on the GPU (Cobra.new_pool / extend_users / generate_users / beam_fusion_users / CobraPool.release):
the fp64 restatement (tests/cobra_generate_reference.py) on each user's concatenated history, the same bits however a history was
split into calls and whichever users share a call or the pool, the paged attention against fp64 at its key-range and page edges,
the null page table against grb_cobra_beam_attention, release and reuse, the page bookkeeping against tests/cobra_pool_reference.py,
and the parameter-version rule."""
import itertools

import pytest
import torch

from tests import cobra_generate_reference as gr
from tests import cobra_params as cp
from tests import cobra_pool_reference as pr
from tests.exact_check import Ledger

pytestmark = pytest.mark.gpu
DEV = "cuda"
# test_cobra_generate_gpu.py's bounds.  score_per_codebook: a score sums one log-probability per codebook, each with the bf16 error of
# its logits through the decoder (measured on an H100 up to 0.020 at C = 1 and 0.031 at C = 3); vec: max-norm relative error of the
# dense vectors (test_cobra_gpu.py's bound); fused: BeamFusion's scores; lead / sim: the fused-score and similarity leads above which
# a rank's item must match
TOL = dict(score_per_codebook=3e-2, vec=3e-2, fused=1e-2, lead=2e-2, sim=5e-3)
LEDGER = Ledger("paged attention against fp64: worst error / allowance")
_error_table = LEDGER.fixture()


def _cfg(C, dh):
    return dict(cp.SMALL, n_codebooks=C, decoder_num_heads=cp.SMALL["d_model"] // dh)


def _model(cfg, seed):
    from genrec_b200.cobra import Cobra
    m = Cobra(**cfg)
    m.load_state_dict(gr.gen_params(cp.cobra_params(cp.shapes(cfg), seed)))
    return m.to(DEV)


def _p64(cfg, seed):
    return {k: (v.double() if v.is_floating_point() else v).to(DEV) for k, v in gr.gen_params(cp.cobra_params(cp.shapes(cfg), seed)).items()}


def _rel(a, ref):
    a, ref = a.double().cpu(), ref.double().cpu()
    return ((a - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()


def _chunk(cfg, ids, text, spans):
    """a padded call from spans (source row, first item, end item): row i holds items lo .. hi-1 of source row src"""
    C, pad = cfg["n_codebooks"], cfg["id_vocab_size"] * cfg["n_codebooks"]
    n = max(1, max(hi - lo for _, lo, hi in spans))
    out = torch.full((len(spans), n * C), pad, dtype=torch.long)
    txt = torch.zeros(len(spans), n, text.shape[2], dtype=torch.long)
    for i, (b, lo, hi) in enumerate(spans):
        out[i, :(hi - lo) * C] = ids[b, lo * C:hi * C]
        txt[i, :hi - lo] = text[b, lo:hi]
    return out.to(DEV), txt.to(DEV)


def _kv_rows(pool, u):
    """every layer's K | V rows of user u, in position order"""
    C, ps = pool.C, pool.page_size
    rows = pr.key_rows(pool.page_table.cpu(), ps, u, pool.lengths[u] * (C + 1))
    return pool.kv.view(pool.kv.shape[0], -1, pool.kv.shape[3])[:, rows]


def _same_model(pool, model):
    assert pool.lengths == model.lengths and pool.free == model.free and pool.pages == model.pages
    assert torch.equal(pool.page_table.cpu(), model.table())


@pytest.mark.parametrize("C,dh,page_size", [(1, 64, 64), (2, 64, 64), (3, 64, 128), (3, 32, 64), (2, 32, 128)])
def test_pool_matches_the_fp64_restatement(C, dh, page_size):
    cfg = _cfg(C, dh)
    m = _model(cfg, 11)
    ids, text = cp.batch(cfg, seed=11)
    pool = m.new_pool(max_users=6, num_pages=40, page_size=page_size)
    users = [4, 0, 5, 2]
    m.extend_users(pool, users, ids.to(DEV), text.to(DEV))
    assert [pool.lengths[u] for u in users] == list(cp.ITEMS)
    for K, T in ((1, 1.0), (7, 0.7)):
        ref = gr.generate(_p64(cfg, 11), cfg, ids.to(DEV), text.to(DEV), K, T)
        settled = [b for b, leads in enumerate(ref["leads"]) if min(leads) > TOL["lead"]]
        assert len(settled) >= 2, ref["leads"]
        out = m.generate_users(pool, users, n_candidates=K, temperature=T)
        for b in settled:
            assert torch.equal(out.sem_ids[b].cpu(), ref["sem_ids"][b].cpu()), b
            assert (out.scores[b].double().cpu() - ref["scores"][b].double().cpu()).abs().max().item() <= TOL["score_per_codebook"] * C, b
            assert _rel(out.dense_vecs[b], ref["dense_vecs"][b]) <= TOL["vec"], b


def test_beam_fusion_users_matches_the_reference():
    cfg = _cfg(3, 64)
    m = _model(cfg, 22)
    ids, text = cp.batch(cfg, items=(20, 20, 20), seed=22)
    pool = m.new_pool(max_users=3, num_pages=12)
    m.extend_users(pool, [0, 1, 2], ids.to(DEV), text.to(DEV))
    ref20 = gr.generate(_p64(cfg, 22), cfg, ids.to(DEV), text.to(DEV), 1)
    vecs, sem = gr.catalog(cfg, ref20["dense_vecs"][:, 0].cpu().float(), 5)
    f = gr.beam_fusion(_p64(cfg, 22), cfg, ids.to(DEV), text.to(DEV), vecs.double().to(DEV), sem.to(DEV), n_candidates=5, n_beam=20)
    out = m.beam_fusion_users(pool, [0, 1, 2], vecs.to(DEV), sem.to(DEV), n_candidates=5, n_beam=20)
    assert (out.scores.double().cpu() - f["scores"].double().cpu()).abs().max().item() <= TOL["fused"]
    lead, sim_lead = f["leads"].cpu(), f["sim_leads"].cpu()
    prev = torch.cat([torch.full_like(lead[:, :1], float("inf")), lead[:, :-1]], dim=1)
    sure = (lead > TOL["lead"]) & (prev > TOL["lead"]) & (sim_lead > TOL["sim"])
    assert bool(sure[:, 0].all())
    assert torch.equal(out.item_ids.cpu()[sure], f["item_ids"].cpu()[sure])
    assert torch.equal(out.sem_ids.cpu()[sure], f["sem_ids"].cpu()[sure])


def _outputs(m, pool, users, vecs, sem):
    g = m.generate_users(pool, users, n_candidates=6)
    f = m.beam_fusion_users(pool, users, vecs, sem, n_candidates=3, n_beam=8)
    return [_kv_rows(pool, u) for u in users], pool.last_hidden[users].clone(), g, f


def _assert_same(a, b, map_b=None):
    """a, b: _outputs of the same users, b's in the order map_b (a's index per b row)"""
    rows = range(len(a[0])) if map_b is None else map_b
    for i, j in enumerate(rows):
        assert torch.equal(a[0][j], b[0][i]), ("kv", j)
        assert torch.equal(a[1][j], b[1][i]), ("last_hidden", j)
        for x, y in ((a[2], b[2]), (a[3], b[3])):
            for fld in x._fields:
                assert torch.equal(getattr(x, fld)[j], getattr(y, fld)[i]), (fld, j)


@pytest.mark.parametrize("C,dh,page_size", [(2, 64, 64), (3, 32, 128), (1, 64, 64)])
def test_a_history_gives_the_same_bits_however_it_was_split(C, dh, page_size):
    cfg = _cfg(C, dh)
    m = _model(cfg, 23)
    items = (1, 2, 7, 20, 13)
    ids, text = cp.batch(cfg, items=items, seed=23)
    oids, otext = cp.batch(cfg, items=(9, 4), seed=24, extra_items=11)   # other users sharing the pool
    g = torch.Generator().manual_seed(23)
    vecs, sem = torch.randn(3000, cfg["d_model"], generator=g).to(DEV), torch.randint(0, 256, (3000, C), generator=g).to(DEV)
    B = len(items)
    kw = dict(max_users=12, num_pages=60, page_size=page_size)
    # one call
    p1 = m.new_pool(**kw)
    model1 = pr.PageModel(12, 60, page_size, C, p1.max_items)
    m.extend_users(p1, list(range(B)), *_chunk(cfg, ids, text, [(b, 0, n) for b, n in enumerate(items)]))
    model1.extend(list(range(B)), list(items))
    _same_model(p1, model1)
    one = _outputs(m, p1, list(range(B)), vecs, sem)
    again = _outputs(m, p1, list(range(B)), vecs, sem)
    _assert_same(one, again)                                        # determinism
    # two calls, different split points, other users in between
    p2 = m.new_pool(**kw)
    model2 = pr.PageModel(12, 60, page_size, C, p2.max_items)
    cut = [0, 1, 3, 11, 5]
    m.extend_users(p2, [7, 6, 5, 4, 3], *_chunk(cfg, ids, text, [(b, 0, cut[b]) for b in range(B)]))   # user 7's row is all pad
    model2.extend([7, 6, 5, 4, 3], cut)
    _same_model(p2, model2)
    m.extend_users(p2, [0, 1], *_chunk(cfg, oids, otext, [(0, 0, 9), (1, 0, 4)]))
    model2.extend([0, 1], [9, 4])
    spans = [(b, cut[b], n) for b, n in enumerate(items)]
    m.extend_users(p2, [7, 6, 5, 4, 3], *_chunk(cfg, ids, text, spans))
    model2.extend([7, 6, 5, 4, 3], [hi - lo for _, lo, hi in spans])
    _same_model(p2, model2)
    _assert_same(one, _outputs(m, p2, [7, 6, 5, 4, 3], vecs, sem))
    # item by item, each step a different subset in a different order, other users interleaved
    p3 = m.new_pool(**kw)
    model3 = pr.PageModel(12, 60, page_size, C, p3.max_items)
    where = [9, 2, 11, 4, 6]
    done = [0] * B
    order = itertools.cycle([[0, 1, 2, 3, 4], [4, 2, 0], [3, 1], [1, 4, 3, 0, 2]])
    step = 0
    while done != list(items):
        rows = [b for b in next(order) if done[b] < items[b]]
        if not rows:
            continue
        users = [where[b] for b in rows]
        spans = [(b, done[b], done[b] + 1) for b in rows]
        if step % 3 == 1:                                           # another user shares the call
            m.extend_users(p3, users + [0], *_chunk(cfg, torch.cat([ids, oids[:1]]), torch.cat([text, otext[:1]]),
                                                    spans + [(B, step // 3 % 9, step // 3 % 9 + 1)]))
            model3.extend(users + [0], [1] * len(rows) + [1])
        else:
            m.extend_users(p3, users, *_chunk(cfg, ids, text, spans))
            model3.extend(users, [1] * len(rows))
        _same_model(p3, model3)
        for b in rows:
            done[b] += 1
        step += 1
    _assert_same(one, _outputs(m, p3, [where[b] for b in (3, 0, 4, 1, 2)], vecs, sem), map_b=[3, 0, 4, 1, 2])


def test_release_and_reuse():
    cfg = _cfg(2, 64)
    m = _model(cfg, 25)
    ids, text = cp.batch(cfg, items=(7, 20), seed=25)
    pool = m.new_pool(max_users=3, num_pages=4)
    model = pr.PageModel(3, 4, 64, 2, pool.max_items)
    m.extend_users(pool, [0, 1], ids.to(DEV), text.to(DEV))
    model.extend([0, 1], [7, 20])
    before = m.generate_users(pool, [0], n_candidates=5)
    pool.release([1])
    model.release([1])
    _same_model(pool, model)
    assert pool.lengths[1] == 0 and not bool(pool.last_hidden[1].any()) and not bool(pool.page_table[1].any())
    m.extend_users(pool, [2], *_chunk(cfg, ids, text, [(1, 0, 20)]))     # the released pages serve another user
    model.extend([2], [20])
    _same_model(pool, model)
    m.extend_users(pool, [1], *_chunk(cfg, ids, text, [(0, 0, 7)]))      # the first user restarts from empty
    model.extend([1], [7])
    _same_model(pool, model)
    fresh = m.new_pool(max_users=3, num_pages=4)
    m.extend_users(fresh, [0], *_chunk(cfg, ids, text, [(0, 0, 7)]))
    pairs = ((m.generate_users(pool, [1], n_candidates=5), m.generate_users(fresh, [0], n_candidates=5)),
             (before, m.generate_users(pool, [0], n_candidates=5)))
    for a, b in pairs:
        for f in a._fields:
            assert torch.equal(getattr(a, f), getattr(b, f)), f
    assert torch.equal(_kv_rows(pool, 1), _kv_rows(fresh, 0)) and torch.equal(pool.last_hidden[1], fresh.last_hidden[0])
    # a chunk beyond max_items or the free pages is refused with the pool unchanged
    snap = (list(pool.lengths), list(pool.free), [list(p) for p in pool.pages], pool.page_table.clone(), pool.kv.clone())
    with pytest.raises(ValueError, match="pages"):                 # two more pages, one free
        m.extend_users(pool, [0, 2], *_chunk(cfg, *cp.batch(cfg, items=(22, 22), seed=26, L=8), [(0, 0, 22), (1, 0, 22)]))
    with pytest.raises(ValueError, match="max_items"):
        m.extend_users(pool, [0], *_chunk(cfg, *cp.batch(cfg, items=(pool.max_items,), seed=26, L=4), [(0, 0, pool.max_items)]))
    assert (pool.lengths, pool.free, pool.pages) == snap[:3]
    assert torch.equal(pool.page_table, snap[3]) and torch.equal(pool.kv, snap[4])


def test_a_pool_written_before_an_optimizer_step_raises():
    cfg = _cfg(3, 64)
    m = _model(cfg, 27)
    ids, text = cp.batch(cfg, items=(3,), seed=27)
    pool = m.new_pool(max_users=2, num_pages=4)
    m.extend_users(pool, [0], ids.to(DEV), text.to(DEV))
    opt = torch.optim.SGD(m.parameters(), lr=0.0)
    for p in m.parameters():
        p.grad = torch.zeros_like(p)
    opt.step()
    with pytest.raises(RuntimeError, match="parameters changed"):
        m.generate_users(pool, [0])
    with pytest.raises(RuntimeError, match="parameters changed"):
        m.extend_users(pool, [1], ids.to(DEV), text.to(DEV))


# ------------------------------------------------------------------------------------------------ kernel stages
def _bf(t):
    return t.to(torch.bfloat16)


@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("page_size", [64, 128])
def test_paged_attention_stage_against_fp64(dh, page_size):
    import genrec_b200.functional as Fn
    g = torch.Generator().manual_seed(dh + page_size)
    H = 2
    D = H * dh
    pages = 16
    model = pr.PageModel(4, pages, page_size, 1, 8192)              # C = 1: two positions per item
    model.extend([1, 0, 3], [40, 20, 10])
    model.release([1])
    model.extend([2, 0, 3], [60, 109, 5])                           # users 0 and 3 hold pages scattered between user 2's
    table = model.table()
    kv = _bf(torch.randn(pages * page_size, 2 * D, generator=g))
    users = [0, 2, 3]
    n_keys = [2 * model.lengths[u] for u in users]                  # 258, 120, 30
    qk = [[1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 258], list(range(1, 121)), [29, 30]]   # edges; a full prefill; one item
    q_off = [0]
    for k in qk:
        q_off.append(q_off[-1] + len(k))
    keys = sum(qk, [])
    R = len(keys)
    for S in (0, 2):
        q = _bf(torch.randn(R, D, generator=g))
        suf = _bf(torch.randn(S, R, 3 * D, generator=g)) if S else None
        anc = torch.randint(0, R, (R, max(S - 1, 0)), generator=g, dtype=torch.int32)
        i32 = lambda x: torch.tensor(x, dtype=torch.int32, device=DEV)
        kvd = kv.to(DEV)
        out = Fn.cobra_paged_attention(q.to(DEV), kvd[:, :D], kvd[:, D:], table.to(DEV), page_size, i32(users), i32(n_keys), max(n_keys),
                                       i32(q_off), i32(keys), H, suf.to(DEV) if S else None, anc.to(DEV) if S > 1 else None, S)
        ref, allow = pr.paged_attention(q, kv[:, :D], kv[:, D:], table, page_size, users, q_off, keys, H, suf, anc, S)
        LEDGER.check(f"dh={dh} ps={page_size} S={S}", [("out", out.cpu(), ref, allow)])


@pytest.mark.parametrize("dh", [32, 64])
def test_paged_beam_attention_gives_the_dense_calls_bits(dh):
    import genrec_b200.functional as Fn
    g = torch.Generator().manual_seed(dh)
    H, B, K, hist = 2, 3, 20, 300
    D = H * dh
    lens = torch.tensor([300, 129, 1], dtype=torch.int32)
    for S in (1, 2):
        hq = _bf(torch.randn(B, hist, 3 * D, generator=g)).to(DEV)
        suf = _bf(torch.randn(S, B * K, 3 * D, generator=g)).to(DEV)
        anc = torch.randint(0, B * K, (B * K, S - 1), generator=g, dtype=torch.int32).to(DEV) if S > 1 else None
        q = suf[S - 1][:, :D]
        dense = Fn.cobra_beam_attention(q, hq, lens.to(DEV), suf, anc, S, H)
        q_off = (torch.arange(B + 1, dtype=torch.int32) * K).to(DEV)
        q_keys = lens.repeat_interleave(K).to(DEV)
        null = Fn.cobra_paged_attention(q, hq[..., D:2 * D], hq[..., 2 * D:], None, hist, None, lens.to(DEV), hist, q_off, q_keys, H, suf, anc, S)
        assert torch.equal(null, dense)
        # the prefill's K | V copied into scattered pages
        model = pr.PageModel(5, 20, 64, 1, 4096)
        model.extend([4, 0, 1, 2, 3], [10, 150, 30, 65, 1])
        model.release([4, 1])
        model.extend([1], [80])
        kv = torch.zeros(20 * 64, 2 * D, dtype=torch.bfloat16, device=DEV)
        for b, u in enumerate((0, 1, 2)):
            kv[model.rows(u, int(lens[b]))] = hq[b, :int(lens[b]), D:]
        users = torch.tensor([0, 1, 2], dtype=torch.int32, device=DEV)
        paged = Fn.cobra_paged_attention(q, kv[:, :D], kv[:, D:], model.table().to(DEV), 64, users, lens.to(DEV), hist, q_off, q_keys, H, suf,
                                         anc, S)
        assert torch.equal(paged, dense)


def test_kv_scatter_writes_each_row_to_its_page():
    import genrec_b200.functional as Fn
    g = torch.Generator().manual_seed(3)
    D = 128
    model = pr.PageModel(3, 10, 64, 2, 4096)
    model.extend([2, 0], [30, 50])
    qkv = _bf(torch.randn(7, 3 * D, generator=g)).to(DEV)
    users, pos = [2, 2, 0, 0, 0, 2, 0], [0, 63, 64, 65, 149, 89, 127]
    kv = torch.zeros(10, 64, 2 * D, dtype=torch.bfloat16, device=DEV)
    Fn.cobra_kv_scatter(qkv, kv, model.table().to(DEV), 64, torch.tensor(users, dtype=torch.int32, device=DEV),
                        torch.tensor(pos, dtype=torch.int32, device=DEV))
    flat = kv.view(-1, 2 * D)
    for r, (u, p) in enumerate(zip(users, pos)):
        assert torch.equal(flat[model.rows(u, p + 1)[p]], qkv[r, D:]), r
    assert int((flat != 0).any(1).sum()) == 7
