"""Every kernel launch of the library checks its own result.  A runtime call that failed earlier in the process leaves its error
behind in the library's CUDA runtime; an entry point whose kernels launched fine must not report that error as its own.  The only
failure made here is a host-side argument error (a device ordinal that does not exist): no kernel faults."""
import pytest
import torch

import genrec_b200.functional as Fn
from genrec_b200 import _lib
from tests.util import make_batch

pytestmark = pytest.mark.gpu

GRB_ENODEV = -3


def _bits(t):
    return t.contiguous().view(torch.uint8)


def test_earlier_runtime_error_is_not_reported_by_a_later_launch():
    from genrec_b200.hstu import HSTULayer
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    T, D, C = 64, 128, 1000
    x = torch.randn(T, D, generator=g).to(dev)
    ln_g, ln_b = (1 + 0.1 * torch.randn(D, generator=g)).to(dev), (0.1 * torch.randn(D, generator=g)).to(dev)
    table = (0.05 * torch.randn(C, D, generator=g)).to(dev)
    tb = table.bfloat16()
    torch.manual_seed(0)
    layer = HSTULayer(64, 2, 0.0, 32, 64, 128, True).to(dev).eval()
    ids, ts, _ = make_batch(3, 40, 50, seed=1)
    xs = torch.randn(3, 40, 64, generator=g).to(dev)
    pad, ts = (ids == 0).to(dev), ts.to(dev)

    def run():
        with torch.no_grad():
            yb, yf, st = Fn.layernorm_fwd(x, ln_g, ln_b, 1e-5, want_bf16=True, want_f32=True)
            logits = Fn.head_logits(x[None], ln_g, ln_b, table, tb, 1e-5)
            y = layer(xs, None, pad, ts)
        return [yb, yf, st, logits, y]

    first = run()
    assert _lib.load().grb_check_device(torch.cuda.device_count() + 5) == GRB_ENODEV
    second = run()
    torch.cuda.synchronize()
    for a, b in zip(first, second):
        assert torch.equal(_bits(a), _bits(b))
