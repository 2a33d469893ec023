"""HSTU attention through the C ABI: bit-exact integer work (time buckets, the bias-index matrix, masks) against the oracle, and
the mma.sync attention core against a plain PyTorch fp32 restatement of the same op on the same bf16 operands."""
import pytest
import torch

from tests.util import relerr

pytestmark = pytest.mark.gpu


def _meta(ids_pad, ts, dev, ntime=64):
    import genrec_b200.functional as Fn
    from genrec_b200.hstu import RelativePositionBias, _thresholds_on
    B, L = ids_pad.shape
    rpb = RelativePositionBias(32, 128, 2)
    return Fn.SeqMeta(ids_pad.to(torch.uint8).to(dev).contiguous(), ts.to(dev).contiguous() if ts is not None else None,
                      rpb.bucket_of_delta(L, dev), _thresholds_on(dev), ntime, 32, rpb.uniform_of(L, dev))


def _oracle_bytes(pad, ts, ntime=64):
    """bucket byte per cell: oracle time bucket where (j <= i and key j not padded), else 64."""
    from oracle import hstu as oh
    B, L = pad.shape
    if ts is not None:
        tb = oh.temporal_bucket(ts.unsqueeze(2) - ts.unsqueeze(1), ntime)
    else:
        tb = torch.zeros(B, L, L, dtype=torch.long)
    ii = torch.arange(L)
    valid = (ii[None, :] <= ii[:, None])[None] & ~pad[:, None, :]
    return torch.where(valid, tb, torch.full_like(tb, 64)).to(torch.uint8)


BOUNDARY = [0, 1, 2, 3, 4, 1022, 1023, 1024, 2044, 2045, 2046, 522823, 522824, 522825, 86400, 2 ** 24 + 1, 10 ** 8, 2 ** 31 - 2,
            2 ** 31 - 1, 2 ** 31, 2 ** 31 + 129, 2 ** 40, 2 ** 62]


@pytest.mark.parametrize("ntime", [64, 20, None], ids=["t64", "t20", "no_ts"])
@pytest.mark.parametrize("L", [1, 33, 130, 200])
def test_bias_index_time_buckets_bit_exact(L, ntime):
    """The bias-index matrix for the timestamp rows below at several lengths, with 64 / 20 time buckets and without timestamps:
    every cell's time bucket and mask == oracle."""
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(L)
    B = 6
    gaps = torch.randint(0, 3 * 86400, (B, L), generator=g)
    gaps[:, ::7] = torch.randint(0, 3, (B, (L + 6) // 7), generator=g)
    ts = 1_300_000_000 + torch.cumsum(gaps, 1)
    # row 1: the boundary differences below 2^31 - 1 against the first event, in order
    narrow = [d for d in BOUNDARY if d < 2 ** 31 - 1]
    for k, d in enumerate(narrow[: max(0, L - 1)]):
        ts[1, k + 1] = ts[1, 0] + d
    ts[1, len(narrow) + 1:] = ts[1, 0] + 2 ** 30
    # row 2: unsorted timestamps (negative differences) ; row 3: every boundary difference (spans >= 2^31 incl. 2^40, 2^62)
    ts[2] = ts[2][torch.randperm(L, generator=g)]
    for k, d in enumerate(BOUNDARY[: max(0, L - 1)]):
        ts[3, k + 1] = ts[3, 0] + d
    # row 4: left padded ; row 5: fully padded ; row 0 keeps a pad in the middle (arbitrary pad positions are legal)
    pad = torch.zeros(B, L, dtype=torch.bool)
    pad[4, : L // 3] = True; ts[4, : L // 3] = 0
    pad[5, :] = True; ts[5, :] = 0
    if L > 5:
        pad[0, 3] = True
    if ntime is None:
        ts = None
    got = (_meta(pad, ts, dev, ntime or 64).bias_index.cpu().to(torch.int32) & 0xFFFF)[:, :, :L]
    want = _oracle_bytes(pad, ts, ntime or 64).to(torch.int32)      # uniform position buckets: index = time bucket, 64 = masked
    bad = got != want
    assert not bad.any(), (bad.nonzero()[:5], got[bad][:5], want[bad][:5])


def test_bias_index_bit_exact():
    """hstu_bias_index_kernel (the attention kernels' [B, L, L] uint16 matrix): time bucket, position bucket and masks == oracle."""
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(3)
    B, L = 5, 70
    ts = 1_300_000_000 + torch.cumsum(torch.randint(0, 86400, (B, L), generator=g), 1)
    for k, d in enumerate(BOUNDARY):
        ts[1, k + 1] = ts[1, 0] + d
    ts[2] = ts[2][torch.randperm(L, generator=g)]
    pad = torch.zeros(B, L, dtype=torch.bool)
    pad[3, :20] = True; ts[3, :20] = 0
    pad[4, :] = True
    m = _meta(pad, ts, dev)
    m.struct()
    got = m.bias_index.cpu().to(torch.int32) & 0xFFFF
    want = _oracle_bytes(pad, ts).to(torch.int32)           # uniform position buckets: index = time bucket, 64 = masked
    assert torch.equal(got[:, :, :L], want)


def _torch_attention(P, zp, dO, pad, ts, H, wpos, wtime, ntime=64):
    """Plain fp32 PyTorch restatement of hstu.py:244-267 on the SAME bf16 operands (P = silu(zp) given), with autograd."""
    from oracle import hstu as oh
    B, L, D4 = P.shape
    D, dh = D4 // 4, D4 // 4 // H
    zp32 = zp.float().requires_grad_(True)
    Pf = torch.nn.functional.silu(zp32)
    # forward operands are the bf16-rounded activations the kernels read
    Pq = Pf + (P.float() - Pf).detach()
    U, V, Q, K = Pq.chunk(4, -1)
    hs = lambda t: t.reshape(B, L, H, dh).transpose(1, 2)
    wpos_ = wpos.clone().requires_grad_(True)
    wtime_ = wtime.clone().requires_grad_(True) if wtime is not None else None
    S = hs(Q) @ hs(K).transpose(-1, -2) + wpos_[0][None, :, None, None]
    if wtime_ is not None and ts is not None:
        tb = oh.temporal_bucket(ts.unsqueeze(2) - ts.unsqueeze(1), ntime).to(P.device)
        S = S + wtime_[tb].permute(0, 3, 1, 2)
    ii = torch.arange(L, device=P.device)
    valid = (ii[None, :] <= ii[:, None])[None, None] & ~pad.to(P.device)[:, None, None, :]
    A = torch.where(valid, torch.nn.functional.silu(S), torch.zeros_like(S))
    O = (A @ hs(V)).transpose(1, 2).reshape(B, L, D)
    O.backward(dO.float())
    return O.detach(), zp32.grad, wpos_.grad, (wtime_.grad if wtime_ is not None else None)


@pytest.mark.parametrize("B,L,D,H,with_ts", [(3, 1, 64, 2, True), (3, 7, 128, 4, True), (4, 64, 128, 4, True), (3, 128, 128, 4, False),
                                             (3, 130, 256, 8, True), (4, 200, 128, 4, True), (3, 257, 64, 2, True), (2, 300, 128, 2, True),
                                             (2, 520, 128, 4, True)])
def test_attention_core_vs_torch_fp32(B, L, D, H, with_ts):
    import genrec_b200.functional as Fn
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(L * 7 + D)
    zp = (0.7 * torch.randn(B, L, 4 * D, generator=g)).to(torch.bfloat16).to(dev)
    P = torch.nn.functional.silu(zp.float()).to(torch.bfloat16)
    dO = (torch.randn(B, L, D, generator=g) / max(1.0, L ** 0.5)).to(torch.bfloat16).to(dev)
    gaps = torch.randint(1, 3 * 86400, (B, L), generator=g)
    gaps[:, ::5] = torch.randint(0, 50, (B, (L + 4) // 5), generator=g)
    ts = 1_300_000_000 + torch.cumsum(gaps, 1)
    pad = torch.zeros(B, L, dtype=torch.bool)
    if B >= 3 and L >= 3:
        pad[1, : L // 3] = True; ts[1, : L // 3] = 0
        pad[2, :] = True; ts[2, :] = 0
    if B >= 4:
        ts[3] = ts[3] * 1000 + torch.arange(L) * (2 ** 33)      # wide path: spans >> 2^31
    wpos = (0.3 * torch.randn(32, H, generator=g)).to(dev)
    wtime = (0.5 * torch.randn(64, H, generator=g)).to(dev) if with_ts else None
    meta = _meta(pad, ts if with_ts else None, dev)
    O = Fn.hstu_attention_fwd(P, meta, H, wpos, wtime)
    dzp, dpos, dtime = Fn.hstu_attention_bwd(P, zp, dO, meta, H, wpos, wtime)
    torch.cuda.synchronize()
    Oref, dzp_ref, dpos_ref, dtime_ref = _torch_attention(P, zp, dO, pad, ts if with_ts else None, H, wpos, wtime)
    valid_rows = ~pad.to(dev)
    assert torch.isfinite(O.float()).all()
    # bf16 rounding of the scores' SiLU (2^-9) and of the outputs is the only difference
    assert relerr(O.float()[valid_rows], Oref[valid_rows]) < 8e-3, relerr(O.float()[valid_rows], Oref[valid_rows])
    assert O.float()[2].abs().max() == 0 if B >= 3 and L >= 3 else True       # fully padded sequence: exact zeros
    D_ = D
    for name, lo in (("V", D_), ("Q", 2 * D_), ("K", 3 * D_)):
        a, r = dzp.float()[..., lo:lo + D_], dzp_ref[..., lo:lo + D_]
        assert relerr(a, r) < 1.5e-2, (name, relerr(a, r))
    assert dzp.float()[..., :D_].abs().max() == 0                             # U columns belong to the gate's backward
    assert relerr(dpos[0], dpos_ref[0]) < 1e-2 and dpos[1:].abs().max() == 0, relerr(dpos[0], dpos_ref[0])
    if with_ts:
        assert relerr(dtime, dtime_ref) < 1e-2, relerr(dtime, dtime_ref)


def test_custom_op_block_equals_module_block():
    """torch.ops.genrec_b200.hstu_layer (dispatcher-registered custom op with a registered autograd formula) == HSTULayer."""
    import genrec_b200.ops  # noqa: F401
    from genrec_b200.hstu import HSTULayer, _thresholds_on
    from tests.util import make_batch
    dev = torch.device("cuda:0")
    torch.manual_seed(1)
    B, L, D, H = 3, 70, 128, 4
    layer = HSTULayer(D, H, 0.0, 32, 64, 128, True).to(dev).train()
    with torch.no_grad():
        for n, p in layer.named_parameters():
            if "attention_bias" in n:
                p.normal_(0, 0.5)
    ids, ts, _ = make_batch(B, L, 50, seed=2)
    ids, ts = ids.to(dev), ts.to(dev)
    x = torch.randn(B, L, D, device=dev)
    dy = torch.randn(B, L, D, device=dev)
    xi = x.clone().requires_grad_(True)
    y = layer(xi, None, ids == 0, ts)
    y.backward(dy)
    ref = (y.detach().clone(), xi.grad.clone(), [p.grad.clone() for p in layer._params()])
    layer.zero_grad(set_to_none=True)
    pad = (ids == 0).to(torch.uint8)
    xj = x.clone().requires_grad_(True)
    y2, _saved = torch.ops.genrec_b200.hstu_layer(xj, pad, ts, _thresholds_on(dev), *layer._params(), H, 64, 0, 0.0, 0, None, 0)
    y2.backward(dy)
    torch.testing.assert_close(y2, ref[0], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(xj.grad, ref[1], rtol=1e-4, atol=1e-5)
    for p, g in zip(layer._params(), ref[2]):
        torch.testing.assert_close(p.grad, g, rtol=2e-3, atol=1e-4 * max(1.0, g.abs().max().item()))
