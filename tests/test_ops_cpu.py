"""torch.ops.genrec_b200.*: schemas are registered and the FakeTensor implementations + autograd wiring trace without a GPU."""
import ctypes

import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode


@pytest.fixture(scope="module", autouse=True)
def lib():
    """The fake implementation of hstu_layer sizes its blob with the library's host-side query."""
    from genrec_b200 import build
    build.build()
    from genrec_b200 import _lib
    return _lib.load()


@pytest.mark.parametrize("D", [64, 128, 256])
def test_fake_saved_blob_matches_the_library(lib, D):
    import genrec_b200.ops  # noqa: F401
    from genrec_b200._lib import HstuDims
    B, L, H = 3, 77, D // 64
    with FakeTensorMode():
        a = _layer_args(B, L, D, H, "cuda")
        _, saved = torch.ops.genrec_b200.hstu_layer(a["x"], a["pad"], a["ts"], a["thr"], *a["params"], H, 64, 0, 0.1, 7, None, 0)
    assert saved.shape == (lib.grb_hstu_layer_saved_bytes(ctypes.byref(HstuDims(B, L, D, H, 32, 64, 0.1, 7, None, 0))),)


def test_ops_are_registered_with_schemas():
    import genrec_b200.ops as ops
    for name in ops.OPS:
        op = getattr(torch.ops.genrec_b200, name)
        assert "Tensor" in str(op.default._schema), name


def _layer_args(B, L, D, H, dev):
    f = lambda *s: torch.empty(*s, device=dev)
    return dict(x=f(B, L, D).requires_grad_(True), pad=torch.empty(B, L, dtype=torch.uint8, device=dev),
                ts=torch.empty(B, L, dtype=torch.int64, device=dev), thr=torch.empty(65, dtype=torch.int64, device=dev),
                params=[f(4 * D, D).requires_grad_(True), f(4 * D).requires_grad_(True), f(32, H).requires_grad_(True),
                        f(64, H).requires_grad_(True), f(D).requires_grad_(True), f(D).requires_grad_(True),
                        f(4 * D, D).requires_grad_(True), f(4 * D).requires_grad_(True), f(D, 4 * D).requires_grad_(True),
                        f(D).requires_grad_(True), f(D).requires_grad_(True), f(D).requires_grad_(True)])


def test_fake_tensor_forward_of_the_block():
    import genrec_b200.ops  # noqa: F401
    B, L, D, H = 3, 50, 128, 4
    with FakeTensorMode():
        a = _layer_args(B, L, D, H, "cuda")
        y, saved = torch.ops.genrec_b200.hstu_layer(a["x"], a["pad"], a["ts"], a["thr"], *a["params"], H, 64, 0, 0.1, 7, None, 0)
        assert y.shape == (B, L, D) and y.device.type == "cuda" and saved.dtype == torch.uint8 and y.requires_grad


def test_meta_forward_and_backward_of_the_block():
    """Shape-only tensors (device "meta", so the autograd engine needs no CUDA context on this box): forward, then backward through
    the registered autograd formula, which itself calls the registered backward op."""
    import genrec_b200.ops  # noqa: F401
    B, L, D, H = 3, 50, 128, 4
    if True:
        a = _layer_args(B, L, D, H, "meta")
        y, saved = torch.ops.genrec_b200.hstu_layer(a["x"], a["pad"], a["ts"], a["thr"], *a["params"], H, 64, 0, 0.1, 7, None, 0)
        assert y.shape == (B, L, D) and y.dtype == torch.float32 and saved.dtype == torch.uint8
        y.sum().backward()
        assert a["x"].grad.shape == (B, L, D)
        for p in a["params"]:
            assert p.grad is not None and p.grad.shape == p.shape
        # without the temporal term
        a = _layer_args(B, L, D, H, "meta")
        a["params"][3] = None
        y, _ = torch.ops.genrec_b200.hstu_layer(a["x"], a["pad"], None, a["thr"], *a["params"], H, 0, 0, 0.0, 0, None, 1)
        y.sum().backward()
        assert a["params"][2].grad.shape == (32, H)


def test_fake_tensor_other_ops():
    import genrec_b200.ops  # noqa: F401
    with FakeTensorMode():
        P = torch.empty(2, 40, 512, dtype=torch.bfloat16, device="cuda")
        pad = torch.empty(2, 40, dtype=torch.uint8, device="cuda")
        ts = torch.empty(2, 40, dtype=torch.int64, device="cuda")
        thr = torch.empty(65, dtype=torch.int64, device="cuda")
        wp, wt = torch.empty(32, 4, device="cuda"), torch.empty(64, 4, device="cuda")
        O = torch.ops.genrec_b200.hstu_attention(P, pad, ts, thr, wp, wt, 4, 0)
        assert O.shape == (2, 40, 128) and O.dtype == torch.bfloat16
        dzp, dpos, dtime = torch.ops.genrec_b200.hstu_attention_backward(P, P, O, pad, ts, thr, wp, wt, 4, 0)
        assert dzp.shape == P.shape and dpos.shape == (32, 4) and dtime.shape == (64, 4)
        ids, emb, res, loss = torch.ops.genrec_b200.rq_residual_argmin(torch.empty(100, 32, device="cuda"), torch.empty(3, 256, 32, device="cuda"), 0.25)
        assert ids.shape == (100, 3) and ids.dtype == torch.int64 and emb.shape == (100, 32, 3) and loss.shape == (100,)
        q = torch.empty(2, 40, 64, dtype=torch.bfloat16, device="cuda")
        out, lse = torch.ops.genrec_b200.sasrec_attention(q, q, q, pad, 2, 0.0, 0, None, 0)
        assert out.shape == q.shape and lse.shape == (2, 2, 40)
        m = torch.ops.genrec_b200.eval_rank_metrics(torch.empty(8, 300, device="cuda"), torch.empty(8, dtype=torch.int64, device="cuda"))
        assert m.shape == (6,)


def test_meta_backward_of_sasrec_attention():
    import genrec_b200.ops  # noqa: F401
    q = torch.empty(2, 40, 64, dtype=torch.bfloat16, device="meta", requires_grad=True)
    pad = torch.empty(2, 40, dtype=torch.uint8, device="meta")
    out, _ = torch.ops.genrec_b200.sasrec_attention(q, q, q, pad, 2, 0.0, 0, None, 0)
    out.float().sum().backward()
    assert q.grad.shape == q.shape


def test_ops_raise_on_cpu_tensors():
    import pytest
    import genrec_b200.ops  # noqa: F401
    with pytest.raises(RuntimeError):
        torch.ops.genrec_b200.rq_residual_argmin(torch.zeros(4, 32), torch.zeros(3, 256, 32), 0.25)
