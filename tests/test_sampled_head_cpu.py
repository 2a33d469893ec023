"""The sampled-softmax head without a GPU: the two C-ABI entry points and their argument checks, the fake kernel and autograd
formula of torch.ops.genrec_b200.head_sampled_loss, the ValueErrors of the modules, and data.sample_negatives."""
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode


@pytest.fixture(scope="module")
def lib():
    from genrec_b200 import build
    build.build()
    from genrec_b200 import _lib
    return _lib.load()


def test_workspace_does_not_grow_with_the_catalog_and_rejects_bad_shapes(lib):
    T = 128 * 200
    small = lib.grb_head_sampled_workspace_bytes(T, 128, 1024)
    assert 0 < small < 64 << 20                     # tens of MB at the benchmark's token count; there is no C argument at all
    assert lib.grb_head_sampled_workspace_bytes(T, 128, 8192) >= small
    for T_, D, N, word in [(T, 256, 64, b"D=256"), (T, 96, 64, b"D=96"), (T, 128, 0, b"N=0"), (T, 128, 8193, b"N=8193"), (0, 128, 64, b"T=0")]:
        assert lib.grb_head_sampled_workspace_bytes(T_, D, N) == 0
        assert word in lib.grb_last_error(), lib.grb_last_error()


def test_argument_checks_come_before_any_launch(lib):
    """every refusal below returns GRB_EINVAL (-1) with a message, on a machine without a GPU"""
    import ctypes
    buf = (ctypes.c_char * 4096)()
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16

    def call(T=8, D=64, C=10, N=4, x=p, negatives=p, dx=p, dtable=p):
        return lib.grb_head_sampled_loss_forward_backward(x, p, p, 1e-5, p, p, negatives, None, T, D, C, N, p, dx, dtable, p, p, p, None)

    for kw, word in [(dict(x=None), b"null"), (dict(negatives=None), b"null"), (dict(D=256), b"D=256"), (dict(N=0), b"N=0"),
                     (dict(N=8193), b"N=8193"), (dict(C=1), b"C=1"), (dict(T=0), b"T=0"), (dict(dtable=None), b"null gradient")]:
        assert call(**kw) == -1, kw
        assert word in lib.grb_last_error(), (kw, lib.grb_last_error())


def test_fake_kernel_and_autograd_formula():
    import genrec_b200.ops as ops
    assert "head_sampled_loss" in ops.OPS
    T, D, C, N = 50, 128, 1000, 64
    with FakeTensorMode():
        f = lambda *s: torch.empty(*s, device="cuda").requires_grad_(True)
        x, g, b, table = f(T, D), f(D), f(D), f(C, D)
        tg = torch.empty(T, dtype=torch.int64, device="cuda")
        neg = torch.empty(N, dtype=torch.int64, device="cuda")
        lq = torch.empty(C, device="cuda")
        for log_q in (lq, None):
            loss, dx, dg, db, dE = torch.ops.genrec_b200.head_sampled_loss(x, g, b, table, tg, neg, log_q, 1e-5)
            assert loss.shape == () and loss.requires_grad and loss.device.type == "cuda"
            assert dx.shape == (T, D) and dg.shape == (D,) and db.shape == (D,) and dE.shape == (C, D)
    # shape-only tensors: backward through the registered formula without a CUDA context
    m = lambda *s: torch.empty(*s, device="meta").requires_grad_(True)
    x, g, b, table = m(T, D), m(D), m(D), m(C, D)
    out = torch.ops.genrec_b200.head_sampled_loss(x, g, b, table, torch.empty(T, dtype=torch.int64, device="meta"),
                                                  torch.empty(N, dtype=torch.int64, device="meta"), None, 1e-5)
    out[0].backward()
    assert x.grad.shape == (T, D) and g.grad.shape == (D,) and b.grad.shape == (D,) and table.grad.shape == (C, D)


def test_op_and_functional_raise_on_cpu_tensors():
    import genrec_b200.ops  # noqa: F401
    with pytest.raises(RuntimeError, match="CUDA"):
        torch.ops.genrec_b200.head_sampled_loss(torch.zeros(4, 64), torch.ones(64), torch.zeros(64), torch.zeros(9, 64),
                                                torch.ones(4, dtype=torch.int64), torch.ones(3, dtype=torch.int64), None, 1e-5)


def test_modules_refuse_negatives_without_targets():
    """the checks come before any device work, so they hold on CPU tensors too"""
    from genrec_b200.hstu import HSTU
    from genrec_b200.sasrec import SASRec
    ids = torch.ones(2, 5, dtype=torch.int64)
    neg = torch.ones(4, dtype=torch.int64)
    hstu = HSTU(20, 5, 64, 2, 1, dropout=0.0)
    sas = SASRec(20, 5, 64, 2, 1, dropout=0.0)
    with pytest.raises(ValueError, match="needs targets"):
        hstu(ids, None, None, negatives=neg)
    with pytest.raises(ValueError, match="needs targets"):
        sas(ids, negatives=neg)
    with pytest.raises(ValueError, match="pass negatives"):
        hstu(ids, None, ids, log_q=torch.zeros(21))
    with pytest.raises(ValueError, match="pass negatives"):
        sas(ids, ids, log_q=torch.zeros(21))


def test_sample_negatives():
    from genrec_b200.data import sample_negatives
    g = torch.Generator().manual_seed(0)
    neg, log_q = sample_negatives(1000, 4096, generator=g)
    assert log_q is None and neg.shape == (4096,) and neg.dtype == torch.int64
    assert int(neg.min()) >= 1 and int(neg.max()) <= 1000 and neg.unique().numel() > 900
    probs = torch.zeros(1001)
    probs[1:11] = torch.arange(1, 11).float()            # only items 1..10 are ever drawn; entry 0 is the padding id
    probs[0] = 5.0
    neg, log_q = sample_negatives(1000, 20000, probs=probs, generator=g)
    assert neg.shape == (20000,) and int(neg.min()) >= 1 and int(neg.max()) <= 10
    assert log_q.shape == (1001,) and log_q.dtype == torch.float32
    torch.testing.assert_close(log_q[1:11].exp(), probs[1:11] / 55.0)
    freq = torch.bincount(neg, minlength=11)[1:11].float() / 20000
    assert (freq - probs[1:11] / 55.0).abs().max().item() < 0.02
    with pytest.raises(ValueError):
        sample_negatives(1000, 8, probs=torch.ones(1000))
    with pytest.raises(ValueError):
        sample_negatives(0, 8)
