"""T5-style attention for TIGER (csrc/attn_t5.cuh + the wgmma projections) against the golden outputs / gradients of the UNMODIFIED
reference module (tests/golden/t5_attention.pt) and, for the attention core alone, against plain fp32 torch on the same bf16-rounded
operands.  Tolerances: bf16 operand level for the module (the reference fixture is fp32), 4e-3 for the core's bf16 outputs, 2e-3 for
its fp32 outputs."""
import math

import pytest
import torch

from tests.util import frob_relerr, relerr

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", ["encoder", "decoder", "cross"])
def test_module_vs_reference_golden(golden, case):
    from genrec_b200.t5_attention import T5Attention
    g = golden("t5_attention.pt")
    c = g["cases"][case]
    dev = torch.device("cuda:0")
    m = T5Attention(g["cfg"]["D"], c["heads"], dropout=0.0, is_cross_attention=c["cross"])
    assert list(m.state_dict().keys()) == list(c["state_dict"].keys())
    m.load_state_dict(c["state_dict"])
    m = m.to(dev).eval()
    x = c["x"].to(dev).requires_grad_(True)
    ctx = c["ctx"].to(dev).requires_grad_(True) if c["cross"] else None
    mask = torch.nn.Transformer.generate_square_subsequent_mask(x.shape[1], device=dev) if c["causal"] else None
    pad = c["pad"].to(dev) if c["pad"] is not None else None
    out, pb = m(x, ctx, ctx, attn_mask=mask, key_padding_mask=pad)
    out.backward(c["dy"].to(dev))
    assert out.dtype == torch.float32 and relerr(out, c["out"]) < 2e-2, relerr(out, c["out"])
    assert frob_relerr(x.grad, c["dx"]) < 3e-2, frob_relerr(x.grad, c["dx"])
    if c["cross"]:
        assert frob_relerr(ctx.grad, c["dctx"]) < 3e-2
        assert pb is None
    else:
        assert pb.shape == (1, c["heads"], x.shape[1], x.shape[1])
    for n, p in m.named_parameters():
        assert frob_relerr(p.grad, c["grads"][n]) < 3e-2, (n, frob_relerr(p.grad, c["grads"][n]))


def _core_reference(Q, K, V, H, bias, bucket, pad, causal, scale):
    B, Lq, D = Q.shape
    Lk, dh = K.shape[1], D // H
    q = Q.view(B, Lq, H, dh).transpose(1, 2); k = K.view(B, Lk, H, dh).transpose(1, 2); v = V.view(B, Lk, H, dh).transpose(1, 2)
    s = (q @ k.transpose(-2, -1)) * scale
    if bias is not None:
        i = torch.arange(Lq)[:, None]; j = torch.arange(Lk)[None, :]
        s = s + bias[:, bucket.long()[(j - i) + Lq - 1]].unsqueeze(0)
    if pad is not None:
        s = s.masked_fill(pad.bool()[:, None, None, :], -1e9)
    if causal:
        s = s + torch.triu(torch.full((Lq, Lk), float("-inf")), diagonal=1)
    return (torch.softmax(s, -1) @ v).transpose(1, 2).reshape(B, Lq, D)


@pytest.mark.parametrize("B,Lq,Lk,H,dh,causal,with_bias,with_pad", [(2, 70, 70, 2, 64, False, True, True), (3, 9, 9, 3, 32, True, True, False),
                                                                     (2, 5, 130, 2, 64, False, False, True), (1, 33, 33, 1, 32, True, True, True)])
def test_attention_core_vs_torch_fp32(B, Lq, Lk, H, dh, causal, with_bias, with_pad):
    from genrec_b200 import t5_attention as t5
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(Lq * 7 + Lk)
    D = H * dh
    rnd = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)          # noqa: E731
    Q, K, V, dO = rnd(B, Lq, D), rnd(B, Lk, D), rnd(B, Lk, D), rnd(B, Lq, D)
    bias = (0.7 * torch.randn(H, 32, generator=g)) if with_bias else None
    bucket = t5.relative_position_buckets(Lq, Lk) if with_bias else None
    pad = None
    if with_pad:
        pad = torch.zeros(B, Lk, dtype=torch.uint8)
        pad[0, Lk - 3:] = 1
        pad[-1, : min(2, Lk - 1)] = 1
    scale = 1 / math.sqrt(dh)
    qf, kf, vf = (t.float().requires_grad_(True) for t in (Q, K, V))
    bf = bias.clone().requires_grad_(True) if with_bias else None
    ref = _core_reference(qf, kf, vf, H, bf, bucket, pad, causal, scale)
    ref.backward(dO.float())
    to = lambda t: t.to(dev) if t is not None else None                         # noqa: E731
    out, lse = t5.attention_core_fwd(to(Q), to(K), to(V), H, to(bias), to(bucket), to(pad), causal, scale)
    dq, dk, dv, dbias = t5.attention_core_bwd(to(Q), to(K), to(V), H, to(bias), to(bucket), to(pad), causal, scale, out, lse, to(dO))
    assert relerr(out, ref) < 6e-3, relerr(out, ref)                            # bf16 output
    assert relerr(dq, qf.grad) < 8e-3, relerr(dq, qf.grad)                      # bf16 output; the saved O is bf16-rounded
    assert relerr(dk, kf.grad) < 8e-3 and relerr(dv, vf.grad) < 6e-3, (relerr(dk, kf.grad), relerr(dv, vf.grad))
    if with_bias:
        assert relerr(dbias, bf.grad) < 8e-3, relerr(dbias, bf.grad)


def test_dropout_mask_is_shared_by_forward_and_backward():
    """V = identity exposes the dropped probability matrix itself: every entry is 0 or P_ij / (1 - p); the backward's dV is built from
    the same matrix."""
    from genrec_b200 import t5_attention as t5
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    B, L, H, dh, p = 2, 48, 1, 64, 0.3
    Q, K = torch.randn(B, L, dh, generator=g).to(torch.bfloat16), torch.randn(B, L, dh, generator=g).to(torch.bfloat16)
    V = torch.zeros(B, L, dh); V[:, torch.arange(L), torch.arange(L)] = 1.0
    V = V.to(torch.bfloat16)
    scale = 1 / math.sqrt(dh)
    P = torch.softmax((Q.float() @ K.float().transpose(1, 2)) * scale, -1)
    out, lse = t5.attention_core_fwd(Q.to(dev), K.to(dev), V.to(dev), H, None, None, None, False, scale, p, 1234, 7)
    Pd = out.float().cpu()[:, :, :L]
    kept = Pd > 0
    frac = 1 - kept.float().mean().item()
    assert abs(frac - p) < 0.04, frac
    torch.testing.assert_close(Pd[kept], (P / (1 - p))[kept], rtol=1.5e-2, atol=1e-4)
    out2, _ = t5.attention_core_fwd(Q.to(dev), K.to(dev), V.to(dev), H, None, None, None, False, scale, p, 1234, 7)
    assert torch.equal(out, out2)                                               # the mask is a function of (seed, site, row, column)
    out3, _ = t5.attention_core_fwd(Q.to(dev), K.to(dev), V.to(dev), H, None, None, None, False, scale, p, 1234, 8)
    assert not torch.equal(out, out3)
    dO = torch.randn(B, L, dh, generator=g).to(torch.bfloat16)
    _, _, dv, _ = t5.attention_core_bwd(Q.to(dev), K.to(dev), V.to(dev), H, None, None, None, False, scale, out, lse, dO.to(dev), p, 1234, 7)
    want = torch.zeros(B, L, dh)
    mask_scale = torch.where(kept, torch.full_like(P, 1 / (1 - p)), torch.zeros_like(P))
    want = (P * mask_scale).transpose(1, 2) @ dO.float()
    assert relerr(dv, want) < 1e-2, relerr(dv, want)


def test_unsupported_masks_raise():
    from genrec_b200.t5_attention import T5Attention
    dev = torch.device("cuda:0")
    m = T5Attention(64, 2).to(dev).eval()
    x = torch.randn(2, 6, 64, device=dev)
    with pytest.raises(NotImplementedError):
        m(x, attn_mask=torch.zeros(6, 6, device=dev))
    with pytest.raises(RuntimeError):
        T5Attention(64, 2)(torch.randn(2, 6, 64))                               # CPU tensors: no fallback
