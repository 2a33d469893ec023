"""grb_head_topk without a GPU: the workspace query, argument refusals before any launch, and the custom op's fake kernel."""
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
    R, D, k = 128, 128, 64
    big = lib.grb_head_topk_workspace_bytes(R, D, 1_000_001, k, 0)
    assert 0 < big < R * 1_000_001 * 4 // 8
    assert lib.grb_head_topk_workspace_bytes(R, D, 10_000_001, k, 0) == big
    assert lib.grb_head_topk_workspace_bytes(R, D, 12_102, 10, 0) > 0
    # the exclusion lists are kept as int32 in the workspace
    assert lib.grb_head_topk_workspace_bytes(R, D, 1_000_001, k, 100) >= big + R * 100 * 4
    for bad in ((0, D, 100, k, 0), (R, 96, 100, k, 0), (R, D, 1, k, 0), (R, D, 100, 0, 0), (R, D, 100, 65, 0), (R, D, 100, k, 16385)):
        assert lib.grb_head_topk_workspace_bytes(*bad) == 0, bad


# fake, never dereferenced device addresses: every case below is refused before anything is touched
_P = 1 << 20


def _call(lib, R=4, D=128, C=100, k=10, E=0, exclude=_P, scores=_P, items=_P):
    return lib.grb_head_topk(_P, _P, _P, ctypes.c_float(1e-5), _P, R, D, C, k, exclude if E else None, E, scores, items, _P, None)


@pytest.mark.parametrize("case,kw,msg", [
    ("k=0", dict(k=0), b"k must"),
    ("k=65", dict(k=65), b"k must"),
    ("D=96", dict(D=96), b"bad shape"),
    ("C=1", dict(C=1), b"bad shape"),
    ("R=0", dict(R=0), b"bad shape"),
    ("E=16385", dict(E=16385), b"exclusion"),
    ("E=-1", dict(E=-1), b"exclusion"),
    ("null exclude", dict(E=5, exclude=None), b"exclude is null"),
    ("null scores", dict(scores=None), b"null argument"),
    ("null items", dict(items=None), b"null argument"),
])
def test_refusals_return_einval_with_a_message(lib, case, kw, msg):
    n0 = lib.grb_launch_count()
    assert _call(lib, **kw) == -1, case
    assert msg in lib.grb_last_error(), (case, lib.grb_last_error())
    assert lib.grb_launch_count() == n0


def test_fake_kernel_shapes(lib):
    import genrec_b200.ops  # noqa: F401
    with FakeTensorMode():
        x = torch.empty(7, 128, device="cuda")
        g = torch.empty(128, device="cuda")
        tb = torch.empty(1001, 128, dtype=torch.bfloat16, device="cuda")
        ex = torch.empty(7, 3, dtype=torch.int64, device="cuda")
        for e in (None, ex):
            s, i = torch.ops.genrec_b200.head_topk(x, g, g, tb, 1e-5, 17, e)
            assert s.shape == (7, 17) and s.dtype == torch.float32
            assert i.shape == (7, 17) and i.dtype == torch.int64


def test_python_argument_checks():
    from genrec_b200 import functional as Fn
    Fn.check_topk_args(1, None, 3, "cpu")
    Fn.check_topk_args(64, torch.zeros(3, 0, dtype=torch.int64), 3, "cpu")
    for k in (0, 65, 2.0, True, None):
        with pytest.raises(ValueError, match="top_k"):
            Fn.check_topk_args(k, None, 3, "cpu")
    for ex, match in ((torch.zeros(3, dtype=torch.int64), r"\[3, E\]"), (torch.zeros(2, 4, dtype=torch.int64), r"\[3, E\]"),
                      (torch.zeros(3, 4, dtype=torch.int32), "int64"), (torch.zeros(3, 16385, dtype=torch.int64), "16384"),
                      ([[1, 2]] * 3, r"\[3, E\]")):
        with pytest.raises(ValueError, match=match):
            Fn.check_topk_args(5, ex, 3, "cpu")
    with pytest.raises(ValueError, match="on cuda"):
        Fn.check_topk_args(5, torch.zeros(3, 4, dtype=torch.int64), 3, "cuda:0")
