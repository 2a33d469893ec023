"""COBRA's paged pool without a GPU: the page bookkeeping model (tests/cobra_pool_reference.py), every host refusal of new_pool /
extend_users / generate_users / beam_fusion_users / release (raised before any library call), the new C entry points refusing bad
arguments, and the fp64 restatement of the paged attention against a direct softmax."""
import ctypes
import os

import pytest
import torch

from tests import cobra_params as cp
from tests import cobra_pool_reference as pr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["grb_cobra_paged_attention", "grb_cobra_paged_attention_workspace_bytes", "grb_cobra_kv_scatter"]


def test_page_model_hands_out_pages_in_row_order_and_reuses_released_ones():
    m = pr.PageModel(max_users=4, num_pages=6, page_size=64, C=3, max_items=40)     # 16 items per page
    m.extend([2, 0], [17, 1])
    assert m.pages[2] == [0, 1] and m.pages[0] == [2] and m.free == [5, 4, 3]
    m.extend([0], [15])                                             # 16 items: still one page
    assert m.pages[0] == [2] and m.lengths[0] == 16
    m.extend([0, 3], [1, 0])
    assert m.pages[0] == [2, 3] and m.lengths[3] == 0 and m.free == [5, 4]
    m.release([2])
    assert m.free == [5, 4, 1, 0] and m.lengths[2] == 0
    m.extend([1], [20])                                             # the released user's first page goes out first
    assert m.pages[1] == [0, 1]
    assert m.table()[1].tolist()[:2] == [0, 1] and m.table()[2].tolist() == [0] * m.cols
    assert m.rows(1, 66)[63:66] == [63, 64, 65]
    assert not m.fits([3], [41]) and not m.fits([3], [33]) and m.fits([3], [32])    # two pages free: 32 items fit, 33 do not


def _pool(cfg, max_users=4, num_pages=8, page_size=64, max_items=None):
    from genrec_b200.cobra import CobraPool
    C = cfg["n_codebooks"]
    max_items = max_items or (cfg["max_len"] - C) // (C + 1)
    return CobraPool(max_users, num_pages, page_size, max_items, cfg["decoder_n_layers"], cfg["d_model"], C, "cpu")


@pytest.fixture
def no_launch(monkeypatch):
    """every functional wrapper fails the test if called"""
    import genrec_b200.functional as Fn

    def boom(name):
        def f(*a, **k):
            raise AssertionError(f"functional.{name} ran before a refusal")
        return f
    for n in dir(Fn):
        if not n.startswith("_") and callable(getattr(Fn, n)) and getattr(getattr(Fn, n), "__module__", "") == Fn.__name__:
            monkeypatch.setattr(Fn, n, boom(n))


def test_new_pool_refusals():
    from genrec_b200.cobra import Cobra
    m = Cobra(**cp.SMALL)
    for kw, msg in ((dict(max_users=0, num_pages=4), "positive"), (dict(max_users=2, num_pages=0), "positive"),
                    (dict(max_users=2, num_pages=4, page_size=96), "multiple of 64"),
                    (dict(max_users=2, num_pages=4, page_size=0), "multiple of 64"),
                    (dict(max_users=2, num_pages=4, max_items=32), "max_items"),          # (128 - 3) // 4 = 31
                    (dict(max_users=2, num_pages=4, max_items=0), "max_items")):
        with pytest.raises(ValueError, match=msg):
            m.new_pool(**kw)
    with pytest.raises(RuntimeError, match="CUDA"):                 # the checks pass: a CPU model cannot hold a pool
        m.new_pool(2, 4, max_items=31)
    # past max_len 8192 + C the paged attention's 8192 history keys bound the default: 8192 // (C+1) = 2048 items at C = 3
    long = Cobra(**dict(cp.SMALL, max_len=20000))
    with pytest.raises(ValueError, match=r"1 \.\. 2048"):
        long.new_pool(2, 4, max_items=2049)
    with pytest.raises(RuntimeError, match="CUDA"):                 # the default passes the checks
        long.new_pool(2, 4)


def test_host_refusals_come_before_any_launch(no_launch):
    from genrec_b200.cobra import Cobra
    cfg = dict(cp.SMALL)
    m = Cobra(**cfg)
    C, V = cfg["n_codebooks"], cfg["id_vocab_size"]
    pool = _pool(cfg, max_items=20, num_pages=3)                    # 16 items per page
    ids, text = cp.batch(cfg, items=(2, 3), L=8)
    with pytest.raises(RuntimeError, match="CUDA"):                 # a valid call stops only at the CUDA requirement
        m.extend_users(pool, [0, 1], ids, text)
    for users, msg in (([0, 4], "out of range"), ([-1, 0], "out of range"), ([1, 1], "distinct"), ([0], "2 rows"), ([], "non-empty")):
        with pytest.raises(ValueError, match=msg):
            m.extend_users(pool, users, ids, text)
    gap = ids.clone()
    gap[1, :C] = V * C
    with pytest.raises(ValueError, match="follows a pad item"):
        m.extend_users(pool, [0, 1], gap, text)
    for c in range(C):                                              # one codebook of one item padded: its rows would not match
        part = ids.clone()
        part[1, C + c] = V * C
        with pytest.raises(ValueError, match="some of its codebooks"):
            m.extend_users(pool, [0, 1], part, text)
    last = ids.clone()
    last[0, :C - 1] = V * C                                         # all but the last codebook padded
    with pytest.raises(ValueError, match="some of its codebooks"):
        m.extend_users(pool, [0, 1], last, text)
    with pytest.raises(ValueError, match="encoder_input_ids"):
        m.extend_users(pool, [0, 1], ids, text[:, :1])
    big, btext = cp.batch(cfg, items=(21,), L=4)
    with pytest.raises(ValueError, match="max_items"):
        m.extend_users(pool, [0], big, btext)
    pool.lengths[2], pool.pages[2], pool.free = 20, [0, 1], [2]     # as if user 2 held 20 items: one page left
    many, mtext = cp.batch(cfg, items=(17, 1), L=4)                 # 17 items need 2 pages
    with pytest.raises(ValueError, match="pages"):
        m.extend_users(pool, [0, 1], many, mtext)
    with pytest.raises(ValueError, match="max_items"):
        m.extend_users(pool, [2], *cp.batch(cfg, items=(1,), L=4))
    assert pool.lengths == [0, 0, 20, 0] and pool.free == [2] and pool.pages[0] == []
    pads = torch.full_like(ids, V * C)
    m.extend_users(pool, [0, 1], pads, torch.zeros_like(text))      # all pad: nothing to do, nothing runs
    assert pool.lengths == [0, 0, 20, 0]
    # generate_users / beam_fusion_users
    vecs, sem = torch.randn(5, cfg["d_model"]), torch.zeros(5, C, dtype=torch.long)
    with pytest.raises(ValueError, match="no item"):
        m.generate_users(pool, [2, 0])
    with pytest.raises(ValueError, match="distinct"):
        m.generate_users(pool, [2, 2])
    with pytest.raises(ValueError, match="out of range"):
        m.generate_users(pool, [9])
    for K in (0, V + 1, 1025):
        with pytest.raises(ValueError, match="n_candidates"):
            m.generate_users(pool, [2], n_candidates=K)
    with pytest.raises(ValueError, match="temperature"):
        m.generate_users(pool, [2], temperature=0.0)
    for nc, nb in ((0, 8), (9, 8)):
        with pytest.raises(ValueError, match="n_candidates"):
            m.beam_fusion_users(pool, [2], vecs, sem, n_candidates=nc, n_beam=nb)
    with pytest.raises(ValueError, match="n_beam"):
        m.beam_fusion_users(pool, [2], vecs, sem, n_candidates=4, n_beam=1025)
    with pytest.raises(ValueError, match="item_sem_ids"):
        m.beam_fusion_users(pool, [2], vecs, sem[:, :2], n_candidates=4, n_beam=8)
    with pytest.raises(ValueError, match="no item"):
        m.beam_fusion_users(pool, [0], vecs, sem, n_candidates=4, n_beam=8)
    with pytest.raises(ValueError, match="distinct"):
        pool.release([1, 1])
    with pytest.raises(ValueError, match="this model"):
        Cobra(**dict(cfg, n_codebooks=2)).extend_users(pool, [0, 1], ids, text)


def test_a_pool_belongs_to_the_parameters_it_was_written_with(no_launch):
    from genrec_b200.cobra import Cobra
    cfg = dict(cp.SMALL)
    m = Cobra(**cfg)
    pool = _pool(cfg)
    pool.param_versions = tuple(p._version for p in m.parameters())
    pool.lengths[0] = 1
    with torch.no_grad():
        m.sparse_head[0].bias.add_(1.0)
    with pytest.raises(RuntimeError, match="parameters changed"):
        m.generate_users(pool, [0])
    with pytest.raises(RuntimeError, match="parameters changed"):
        m.extend_users(pool, [0], *cp.batch(cfg, items=(1,), L=4))


def test_new_symbols_are_declared_and_bound():
    from genrec_b200 import _lib
    header = open(os.path.join(ROOT, "include", "genrec_b200.h")).read()
    for n in NAMES:
        assert n + "(" in header and n in _lib.SIGNATURES, n


def test_entry_points_refuse_bad_arguments_before_any_launch():
    from genrec_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("the library is not built")
    lib = _lib.load()
    x = ctypes.c_void_p(256)                                        # never dereferenced: every call below is refused
    i32 = ctypes.c_void_p(512)
    assert lib.grb_cobra_paged_attention_workspace_bytes(4, 2, 48, 100) == 0
    assert lib.grb_cobra_paged_attention_workspace_bytes(4, 2, 64, 8193) == 0
    assert lib.grb_cobra_paged_attention_workspace_bytes(0, 2, 64, 100) == 0
    assert lib.grb_cobra_paged_attention_workspace_bytes(4, 2, 64, 129) == 4 * 2 * 2 * 66 * 4

    def attn(**kw):
        a = dict(q=x, ldq=384, k=x, v=x, ld_kv=256, pt=i32, pt_ld=4, ps=64, users=i32, hist=i32, max_keys=100, q_off=i32, q_keys=i32, R=4,
                 sk=None, sv=None, ld_suf=384, stride=0, anc=None, S=0, B=2, H=2, dh=64, out=x, ldo=128, ws=x)
        a.update(kw)
        return lib.grb_cobra_paged_attention(*a.values(), None)
    for kw, msg in ((dict(q=None), "null"), (dict(q_keys=None), "null"), (dict(q_off=None), "null"), (dict(hist=None), "null"),
                    (dict(ws=None), "null"), (dict(ps=96), "multiple of 64"), (dict(ps=0), "multiple of 64"), (dict(dh=48), "head_dim"),
                    (dict(pt_ld=1), "cannot hold"), (dict(pt=None, ps=64), "below max_keys"), (dict(S=1), "suffix"),
                    (dict(S=2, sk=x, sv=x, stride=4 * 384), "anc"), (dict(max_keys=8193, pt_ld=200), "hist_rows"), (dict(R=0), "R=0")):
        assert attn(**kw) != 0, kw
        assert msg in _lib.last_error(), (kw, _lib.last_error())

    def scatter(**kw):
        a = dict(qkv=x, ld=384, R=4, D=128, pt=i32, pt_ld=4, ps=64, ru=i32, rp=i32, kv=x)
        a.update(kw)
        return lib.grb_cobra_kv_scatter(*a.values(), None)
    for kw, msg in ((dict(qkv=None), "null"), (dict(pt=None), "null"), (dict(rp=None), "null"), (dict(kv=None), "null"),
                    (dict(ps=32), "multiple of 64"), (dict(D=12), "D=12"), (dict(ld=200), "ld_qkv"), (dict(R=0), "R=0")):
        assert scatter(**kw) != 0, kw
        assert msg in _lib.last_error(), (kw, _lib.last_error())


@pytest.mark.parametrize("dh", [32, 64])
def test_paged_attention_restatement_matches_a_dense_softmax(dh):
    g = torch.Generator().manual_seed(dh)
    H, page_size = 2, 64
    D = H * dh
    model = pr.PageModel(max_users=3, num_pages=12, page_size=page_size, C=1, max_items=200)
    model.extend([1, 0], [40, 10])
    model.release([1])
    model.extend([2, 0], [70, 25])                                  # user 0's pages are scattered between user 2's
    table = model.table()
    k = torch.randn(12 * page_size, D, generator=g, dtype=torch.float64)
    v = torch.randn(12 * page_size, D, generator=g, dtype=torch.float64)
    users = [2, 0]
    hist = [140, 70]
    q_keys = [1, 63, 64, 65, 128, 129, 140] + [70, 1, 2]
    q_off = [0, 7, 10]
    q = torch.randn(10, D, generator=g, dtype=torch.float64)
    out, allow = pr.paged_attention(q, k, v, table, page_size, users, q_off, q_keys, H)
    for b, u in enumerate(users):
        for r in range(q_off[b], q_off[b + 1]):
            rows = model.rows(u, q_keys[r])
            assert torch.allclose(out[r], pr.dense_softmax(q[r], k[rows], v[rows], H), rtol=0, atol=1e-12)
    assert bool((allow > 0).all()) and max(hist) <= model.lengths[2] * 2
    # a null page table: user b's keys are rows b page_size ..
    out2, _ = pr.paged_attention(q[:2], k, v, None, 100, None, [0, 1, 2], [5, 100], H)
    assert torch.allclose(out2[1], pr.dense_softmax(q[1], k[100:200], v[100:200], H), rtol=0, atol=1e-12)
