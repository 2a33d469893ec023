"""FlatAdam(lazy_table=True) without a GPU: an fp64 restatement of the lazy rule, checked against torch.optim.SparseAdam (eps = 0,
where SparseAdam's form and FlatAdam's coincide) and against a dense torch.optim.Adam run whose rows are all touched at every step;
the argument checks of the three C-ABI entry points; and the ValueErrors of the optimizer's constructor.
tests/test_lazy_table_gpu.py checks the kernels against the same restatement (hstu_block_reference.lazy_adam_reference)."""
import ctypes

import pytest
import torch

from tests.hstu_block_reference import lazy_adam_reference


def test_reference_matches_sparse_adam_at_eps_zero():
    C, D, lr, betas = 40, 8, 1e-2, (0.9, 0.99)
    gen = torch.Generator().manual_seed(0)
    w0 = torch.randn(C, D, dtype=torch.float64, generator=gen)
    param = torch.nn.Parameter(w0.clone())
    # SparseAdam refuses eps = 0; next to the sqrt(v) of these gradients, 1e-30 moves no fp64 digit the comparison looks at
    sparse = torch.optim.SparseAdam([param], lr=lr, betas=betas, eps=1e-30)
    p, m, v = w0.clone(), torch.zeros(C, D, dtype=torch.float64), torch.zeros(C, D, dtype=torch.float64)
    for step in range(1, 7):
        rows = torch.randperm(C, generator=gen)[:5 + 3 * step]            # a different row set every step
        gvals = torch.randn(len(rows), D, dtype=torch.float64, generator=gen)
        dense_g = torch.zeros(C, D, dtype=torch.float64)
        dense_g[rows] = gvals
        param.grad = torch.sparse_coo_tensor(rows[None], gvals, (C, D)).coalesce()
        sparse.step()
        p, m, v = lazy_adam_reference(p, dense_g, m, v, rows.tolist(), step, lr, betas, 0.0, 0.0)
        torch.testing.assert_close(p, param.detach(), rtol=1e-12, atol=1e-12)
        st = sparse.state[param]
        torch.testing.assert_close(m, st["exp_avg"], rtol=1e-12, atol=1e-14)
        torch.testing.assert_close(v, st["exp_avg_sq"], rtol=1e-12, atol=1e-14)


def test_reference_touching_every_row_is_dense_adam():
    C, D, lr, betas, eps, wd = 30, 8, 1e-2, (0.9, 0.98), 1e-3, 0.05
    gen = torch.Generator().manual_seed(1)
    w0 = torch.randn(C, D, dtype=torch.float64, generator=gen)
    param = torch.nn.Parameter(w0.clone())
    dense = torch.optim.Adam([param], lr=lr, betas=betas, eps=eps, weight_decay=wd)
    p, m, v = w0.clone(), torch.zeros(C, D, dtype=torch.float64), torch.zeros(C, D, dtype=torch.float64)
    for step in range(1, 7):
        g = torch.randn(C, D, dtype=torch.float64, generator=gen)
        param.grad = g.clone()
        dense.step()
        p, m, v = lazy_adam_reference(p, g, m, v, range(C), step, lr, betas, eps, wd)
        torch.testing.assert_close(p, param.detach(), rtol=1e-12, atol=1e-12)
        torch.testing.assert_close(m, dense.state[param]["exp_avg"], rtol=1e-12, atol=1e-14)


def test_reference_leaves_untouched_rows_alone():
    gen = torch.Generator().manual_seed(2)
    p, g, m, v = (torch.randn(12, 4, generator=gen) for _ in range(4))
    v = v.abs()
    p2, m2, v2 = lazy_adam_reference(p, g, m, v, [3, 7, 3], 4, 1e-2, (0.9, 0.999), 1e-8, 0.01)
    keep = [i for i in range(12) if i not in (3, 7)]
    for new, old in ((p2, p), (m2, m), (v2, v)):
        assert torch.equal(new[keep], old[keep].double())
        assert not torch.equal(new[[3, 7]], old[[3, 7]].double())


@pytest.fixture(scope="module")
def lib():
    from genrec_b200 import build
    build.build()
    from genrec_b200 import _lib
    return _lib.load()


def test_argument_checks_come_before_any_launch(lib):
    """every refusal below returns GRB_EINVAL (-1) with a message, on a machine without a GPU"""
    buf = (ctypes.c_char * 4096)()
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16

    def mark(ids=p, n=8, C=10, flag=p, rows=p, count=p):
        return lib.grb_rowset_mark(ids, n, C, flag, rows, count, None)

    for kw, word in [(dict(ids=None), b"null"), (dict(flag=None), b"null"), (dict(rows=None), b"null"), (dict(count=None), b"null"),
                     (dict(C=1), b"C=1")]:
        assert mark(**kw) == -1, kw
        assert word in lib.grb_last_error(), (kw, lib.grb_last_error())
    assert lib.grb_rowset_mark_all(None, None) == -1 and b"null" in lib.grb_last_error()

    def step(pp=p, g=p, m=p, v=p, mirror=p, n=1024, off=0, C=8, D=64, flag=p, rows=p, count=p, all_word=p, state=p):
        return lib.grb_adam_step_lazy_table(pp, g, m, v, mirror, n, off, C, D, flag, rows, count, all_word, state, 1e-3, 0.9, 0.999, 1e-8,
                                            0.0, 1.0, None)

    cases = [(dict(pp=None), b"null"), (dict(g=None), b"null"), (dict(m=None), b"null"), (dict(v=None), b"null"),
             (dict(mirror=None), b"null"), (dict(flag=None), b"null"), (dict(rows=None), b"null"), (dict(count=None), b"null"),
             (dict(all_word=None), b"null"), (dict(state=None), b"null"), (dict(C=1), b"C=1"), (dict(D=62), b"D=62"),
             (dict(D=96), b"D=96"), (dict(off=1024 - 8 * 64 + 4), b"outside"), (dict(n=8 * 64 - 1), b"outside"),
             (dict(off=2), b"aligned")]
    for kw, word in cases:
        assert step(**kw) == -1, kw
        assert word in lib.grb_last_error(), (kw, lib.grb_last_error())


class _Pair(torch.nn.Module):
    def __init__(self, a, b):
        super().__init__()
        self.a, self.b = a, b


def test_constructor_refuses_what_it_does_not_cover(monkeypatch):
    """the refusals come before any device work, so they run on the CPU"""
    from genrec_b200 import optim
    from genrec_b200.hstu import HSTU
    h = HSTU(20, 8, 64, 2, 1, dropout=0.0)
    for model, word in [(torch.nn.Linear(4, 4), "exactly one HSTU"), (_Pair(h, HSTU(20, 8, 64, 2, 1, dropout=0.0)), "exactly one HSTU")]:
        with pytest.raises(ValueError, match=word):
            optim.FlatAdam(model, lazy_table=True)
    with pytest.raises(ValueError, match="grad_sink"):
        optim.FlatAdam(h, lazy_table=True, grad_sink=False)
    monkeypatch.setattr(optim, "world_size", lambda group=None: 2)
    with pytest.raises(ValueError, match="one process"):
        optim.FlatAdam(h, lazy_table=True)
