"""grb_head_rank without a GPU: the ABI symbols, the workspace query, argument refusals before any launch, and the custom op's fake
kernel."""
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


def test_symbols_resolve(lib):
    so = ctypes.CDLL(lib._name)
    for name in ("grb_head_rank", "grb_head_rank_workspace_bytes"):
        assert hasattr(so, name), name


def test_workspace_grows_with_rows_and_exclusions_not_with_the_catalog(lib):
    R, D = 128, 128
    small = lib.grb_head_rank_workspace_bytes(R, D, 12_102, 0)
    assert 0 < small
    assert lib.grb_head_rank_workspace_bytes(R, D, 10_000_001, 0) == small
    assert lib.grb_head_rank_workspace_bytes(R, D, 1_000_001, 0) == small
    assert lib.grb_head_rank_workspace_bytes(2 * R, D, 12_102, 0) > small
    assert lib.grb_head_rank_workspace_bytes(1024, D, 10_000_001, 0) < 1024 * 10_000_001 * 4 // 1000
    # the exclusion lists are kept sorted as int32 in the workspace
    with_ex = lib.grb_head_rank_workspace_bytes(R, D, 12_102, 100)
    assert with_ex >= small + R * 100 * 4
    assert lib.grb_head_rank_workspace_bytes(R, D, 12_102, 200) > with_ex
    assert lib.grb_head_rank_workspace_bytes(R, D, 10_000_001, 100) == with_ex
    for bad in ((0, D, 100, 0), (R, 96, 100, 0), (R, D, 1, 0), (R, D, 100, 16385), (R, D, 100, -1)):
        assert lib.grb_head_rank_workspace_bytes(*bad) == 0, bad


# fake, never dereferenced device addresses: every case below is refused before anything is touched
_P = 1 << 20


def _call(lib, R=4, D=128, C=100, E=0, x=_P, table=_P, targets=_P, exclude=_P, metrics=_P, ranks=_P):
    return lib.grb_head_rank(x, _P, _P, ctypes.c_float(1e-5), table, R, D, C, targets, exclude if E else None, E, metrics, ranks, _P,
                             None)


@pytest.mark.parametrize("case,kw,msg", [
    ("D=96", dict(D=96), b"D=96"),
    ("D=32", dict(D=32), b"D=32"),
    ("C=1", dict(C=1), b"C=1"),
    ("C=0", dict(C=0), b"C=0"),
    ("R=0", dict(R=0), b"R=0"),
    ("E=16385", dict(E=16385), b"E=16385"),
    ("E=-1", dict(E=-1), b"E=-1"),
    ("null x", dict(x=None), b"x is null"),
    ("null table", dict(table=None), b"table_bf16 is null"),
    ("null targets", dict(targets=None), b"targets is null"),
    ("null exclude", dict(E=5, exclude=None), b"exclude is null"),
    ("nothing to write", dict(metrics=None, ranks=None), b"metrics and ranks"),
])
def test_refusals_return_einval_with_a_message(lib, case, kw, msg):
    n0 = lib.grb_launch_count()
    assert _call(lib, **kw) == -1, case
    assert msg in lib.grb_last_error(), (case, lib.grb_last_error())
    assert lib.grb_launch_count() == n0


def test_fake_kernel_shapes(lib):
    import genrec_b200.ops as ops
    assert "head_rank_metrics" in ops.OPS
    with FakeTensorMode():
        x = torch.empty(7, 128, device="cuda")
        g = torch.empty(128, device="cuda")
        tb = torch.empty(1001, 128, dtype=torch.bfloat16, device="cuda")
        tg = torch.empty(7, dtype=torch.int64, device="cuda")
        ex = torch.empty(7, 3, dtype=torch.int64, device="cuda")
        for e in (None, ex):
            m, r = torch.ops.genrec_b200.head_rank_metrics(x, g, g, tb, 1e-5, tg, e)
            assert m.shape == (6,) and m.dtype == torch.float32
            assert r.shape == (7,) and r.dtype == torch.int32


def test_python_argument_checks():
    from genrec_b200 import functional as Fn
    Fn.check_exclude_arg(None, 3, "cpu")
    Fn.check_exclude_arg(torch.zeros(3, 0, dtype=torch.int64), 3, "cpu")
    for ex, match in ((torch.zeros(3, dtype=torch.int64), r"\[3, E\]"), (torch.zeros(3, 4, dtype=torch.int32), "int64"),
                      (torch.zeros(3, 16385, dtype=torch.int64), "16384")):
        with pytest.raises(ValueError, match=match):
            Fn.check_exclude_arg(ex, 3, "cpu")
