"""grb_head_candidates without a GPU: the workspace query, argument refusals before any launch, the custom op's fake kernel and the
Python argument checks of Fn.head_candidates, retrieve and the num_candidates keyword of extend / extend_users."""
import ctypes

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode


@pytest.fixture(scope="module")
def lib():
    from genrec_b200 import build
    build.build()
    from genrec_b200 import _lib
    return _lib.load()


def test_workspace_does_not_grow_with_the_catalog(lib):
    R, D = 128, 128
    for k in (65, 500, 2048):
        big = lib.grb_head_candidates_workspace_bytes(R, D, 1_000_001, k, 0)
        assert 0 < big < R * 1_000_001 * 4 // 8
        assert lib.grb_head_candidates_workspace_bytes(R, D, 10_000_001, k, 0) == big
        # the exclusion lists are kept as int32 in the workspace
        assert lib.grb_head_candidates_workspace_bytes(R, D, 1_000_001, k, 100) >= big + R * 100 * 4
    # k <= 64 runs the top-k head, with its workspace
    for k in (1, 10, 64):
        assert lib.grb_head_candidates_workspace_bytes(R, D, 1_000_001, k, 7) == lib.grb_head_topk_workspace_bytes(R, D, 1_000_001, k, 7)


def test_workspace_grows_with_rows_times_k(lib):
    C, D = 1_000_001, 128
    w = {(R, k): lib.grb_head_candidates_workspace_bytes(R, D, C, k, 0) for R in (128, 1024) for k in (256, 2048)}
    # the collect buffer alone holds 4 k (score, id) pairs per row
    assert w[128, 2048] - w[128, 256] >= 128 * 4 * (2048 - 256) * 8
    assert w[1024, 2048] - w[1024, 256] >= 1024 * 4 * (2048 - 256) * 8
    assert w[1024, 2048] >= 8 * 128 * 4 * 2048 * 8


def test_workspace_refusals(lib):
    R, D, k = 128, 128, 500
    for bad in ((0, D, 100, k, 0), (R, 96, 100, k, 0), (R, D, 1, k, 0), (R, D, 100, 0, 0), (R, D, 100, 2049, 0), (R, D, 100, k, 16385),
                (R, D, 100, k, -1)):
        assert lib.grb_head_candidates_workspace_bytes(*bad) == 0, bad


# fake, never dereferenced device addresses: every case below is refused before anything is touched
_P = 1 << 20


def _call(lib, R=4, D=128, C=100, k=500, E=0, exclude=_P, scores=_P, items=_P):
    return lib.grb_head_candidates(_P, _P, _P, ctypes.c_float(1e-5), _P, R, D, C, k, exclude if E else None, E, scores, items, _P, None)


@pytest.mark.parametrize("case,kw,msg", [
    ("k=0", dict(k=0), b"k must lie in [1, 2048]"),
    ("k=-3", dict(k=-3), b"k must lie in [1, 2048]"),
    ("k=2049", dict(k=2049), b"k must lie in [1, 2048]"),
    ("D=96", dict(D=96), b"bad shape"),
    ("C=1", dict(C=1), b"bad shape"),
    ("R=0", dict(R=0), b"bad shape"),
    ("E=16385", dict(E=16385), b"exclusion"),
    ("E=-1", dict(E=-1), b"exclusion"),
    ("null exclude", dict(E=5, exclude=None), b"exclude is null"),
    ("null exclude, k=10", dict(k=10, E=5, exclude=None), b"exclude is null"),
    ("null scores", dict(scores=None), b"null argument"),
    ("null items", dict(items=None), b"null argument"),
])
def test_refusals_return_einval_with_a_message(lib, case, kw, msg):
    n0 = lib.grb_launch_count()
    assert _call(lib, **kw) == -1, case
    assert msg in lib.grb_last_error(), (case, lib.grb_last_error())
    assert lib.grb_launch_count() == n0


def test_fake_kernel_shapes(lib):
    import genrec_b200.ops as ops
    assert "head_candidates" in ops.OPS
    with FakeTensorMode():
        x = torch.empty(7, 128, device="cuda")
        g = torch.empty(128, device="cuda")
        tb = torch.empty(100_001, 128, dtype=torch.bfloat16, device="cuda")
        ex = torch.empty(7, 3, dtype=torch.int64, device="cuda")
        for k in (5, 500, 2048):
            for e in (None, ex):
                s, i = torch.ops.genrec_b200.head_candidates(x, g, g, tb, 1e-5, k, e)
                assert s.shape == (7, k) and s.dtype == torch.float32
                assert i.shape == (7, k) and i.dtype == torch.int64


def test_python_argument_checks():
    from genrec_b200 import functional as Fn
    assert Fn.CANDIDATES_MAX_K == 2048
    Fn.check_candidates_args(1, None, 3, "cpu")
    Fn.check_candidates_args(2048, torch.zeros(3, 0, dtype=torch.int64), 3, "cpu")
    for k in (0, 2049, -1, 500.0, True, None):
        with pytest.raises(ValueError, match="num_candidates"):
            Fn.check_candidates_args(k, None, 3, "cpu")
    for ex, match in ((torch.zeros(3, dtype=torch.int64), r"\[3, E\]"), (torch.zeros(2, 4, dtype=torch.int64), r"\[3, E\]"),
                      (torch.zeros(3, 4, dtype=torch.int32), "int64"), (torch.zeros(3, 16385, dtype=torch.int64), "16384"),
                      ([[1, 2]] * 3, r"\[3, E\]")):
        with pytest.raises(ValueError, match=match):
            Fn.check_candidates_args(500, ex, 3, "cpu")
    with pytest.raises(ValueError, match="on cuda"):
        Fn.check_candidates_args(500, torch.zeros(3, 4, dtype=torch.int64), 3, "cuda:0")


def _hstu():
    from genrec_b200.hstu import HSTU
    return HSTU(97, 20, 64, 2, 1, dropout=0.0).eval()


def test_serving_keywords_are_checked_before_any_work():
    m = _hstu()
    ex = torch.zeros(3, 4, dtype=torch.int64)
    for kw, match in ((dict(top_k=10, num_candidates=500), "not both"), (dict(top_k=10, num_candidates=500, exclude=ex), "not both"),
                      (dict(exclude=ex), "top_k"), (dict(num_candidates=0), "num_candidates"),
                      (dict(num_candidates=2049), "num_candidates"), (dict(num_candidates=500, exclude=ex[:2]), r"\[3, E\]")):
        for what in ("extend", "extend_users"):
            with pytest.raises(ValueError, match=match):
                m._check_serving_topk(what, kw.get("top_k"), kw.get("num_candidates"), kw.get("exclude"), 3, "cpu")
    m._check_serving_topk("extend", None, 2048, ex, 3, "cpu")
    m._check_serving_topk("extend", 64, None, ex, 3, "cpu")
    m._check_serving_topk("extend", None, None, None, 3, "cpu")


def test_retrieve_refuses_fp32_and_bad_counts():
    m = _hstu()
    ids = torch.ones(3, 20, dtype=torch.int64)
    for k in (0, 2049, 2.0):
        with pytest.raises(ValueError, match="num_candidates"):
            m.retrieve(ids, num_candidates=k)
    m.set_precision("fp32")
    with pytest.raises(RuntimeError, match="bf16"):
        m.retrieve(ids, num_candidates=500)
    with pytest.raises(RuntimeError, match="bf16"):
        m._check_serving_topk("extend", None, 500, None, 3, "cpu")
