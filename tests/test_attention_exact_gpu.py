"""The SASRec and T5 attention cores against the fp64 references of tests/attention_reference.py, at their tile edges, padding edges
and dropout rates; the T5 backward's reproducibility; and the values of the FFN's d-activation GEMM.  `pytest -s` prints each case's
worst and Frobenius ratios (error over the per-element allowance)."""
import math

import pytest
import torch

from tests import attention_reference as ar

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _report(tag, err):
    print(f"{tag}: {ar.fmt(err)}")


# ------------------------------------------------------------------------------------------------ SASRec
SAS_L = [1, 2, 17, 63, 64, 65, 127, 128, 129, 200, 513]
SAS_CASES = [(L, dh, (1, 2, 4)[n % 3], (0.0, 0.2, 0.5)[(n + k) % 3]) for k, dh in enumerate((32, 64)) for n, L in enumerate(SAS_L)]


def _sas_inputs(B, L, H, dh, seed):
    """Scores spanning about +-30 (q ~ 8 N(0, 1)); past the first key tile one key per sequence is scaled up so the running maximum
    of many rows first appears in a later tile.  Padding: left (row 0), a hole in the middle plus tail (row 1), exactly one valid
    token (row 2), a fully padded sequence (row 3), none (row 4)."""
    g = torch.Generator().manual_seed(seed)
    D = H * dh
    Q = 8 * torch.randn(B, L, D, generator=g)
    K = torch.randn(B, L, D, generator=g)
    if L > 64:
        K[:, 64 + (L - 64) // 2] *= 3
    V, dO = torch.randn(B, L, D, generator=g), torch.randn(B, L, D, generator=g)
    pad = torch.zeros(B, L, dtype=torch.uint8)
    pad[0, : (L + 1) // 3] = 1
    pad[1, L // 3: L // 3 + max(1, L // 5)] = 1
    pad[1, L - max(1, L // 7):] = 1
    pad[2] = 1
    pad[2, L // 2] = 0
    pad[3] = 1
    return [t.bfloat16().to(DEV) for t in (Q, K, V, dO)] + [pad.to(DEV)]


@pytest.mark.parametrize("L,dh,H,p", SAS_CASES)
def test_sasrec_core_vs_fp64(L, dh, H, p):
    import genrec_b200.functional as Fn
    B, seed, layer = 5, 1000 + L, 1
    Q, K, V, dO, pad = _sas_inputs(B, L, H, dh, L * 7 + dh)
    out, lse = Fn.sasrec_attention_fwd(Q, K, V, pad, H, p, seed, None, layer)
    dq, dk, dv = Fn.sasrec_attention_bwd(Q, K, V, pad, out, lse, dO, H, p, seed, None, layer)
    ref = ar.sasrec_reference(Q, K, V, pad, H, dO, out, p, seed, layer)
    got = {"out": out, "dq": dq, "dk": dk, "dv": dv, "lse": lse}
    err = ar.errors(got, ref, ("out", "dq", "dk", "dv"))
    _report(f"sasrec L={L} dh={dh} H={H} p={p}", err)
    assert not ar.violations(err, "sas"), ar.fmt(err)
    assert not ar.sasrec_exact(got, ref)
    live = ref["valid"].any(-1)
    d = (lse.double() - ref["lse"])[live].abs()
    assert d.numel() == 0 or d.max().item() <= 1e-4 * (1 + ref["lse"][live].abs().max().item())


@pytest.mark.parametrize("dh,H,p", [(32, 2, 0.2), (64, 1, 0.5), (64, 2, 0.2)])
def test_sasrec_dropout_pattern_is_the_restated_mask(dh, H, p):
    """V = identity per head exposes the dropped probability matrix: O_ij = 0 exactly where the restated mask drops (i, j) among
    the cells that take part in the softmax (scores kept small, so no kept probability underflows)."""
    import genrec_b200.functional as Fn
    B, L, seed, layer = 3, dh, 77, 2
    g = torch.Generator().manual_seed(dh + H)
    D = H * dh
    Q, K = (0.5 * torch.randn(B, L, D, generator=g)).bfloat16(), (0.5 * torch.randn(B, L, D, generator=g)).bfloat16()
    V = torch.zeros(B, L, D)
    for h in range(H):
        V[:, torch.arange(L), h * dh + torch.arange(L)] = 1.0
    pad = torch.zeros(B, L, dtype=torch.uint8)
    pad[1, :5] = 1
    pad[2, 7:11] = 1
    out, _ = Fn.sasrec_attention_fwd(Q.to(DEV), K.to(DEV), V.bfloat16().to(DEV), pad.to(DEV), H, p, seed, None, layer)
    Pd = out.float().cpu().view(B, L, H, dh).transpose(1, 2)                 # [B, H, i, j]
    ref = ar.sasrec_reference(Q, K, V.bfloat16(), pad, H, p=p, seed=seed, layer=layer)
    valid = ref["valid"]
    assert torch.equal((Pd == 0)[valid], ref["drop"][valid])
    assert not bool((Pd[~valid] != 0).any())


# ------------------------------------------------------------------------------------------------ T5
T5_LQ = [1, 4, 30, 31, 32, 33, 61, 64, 65, 130]
T5_LK = [1, 4, 61, 63, 64, 65, 129, 200]
T5_CASES = [(lq, lk, (32, 64)[n % 2], n % 3 != 2, n % 4 != 3, (0.0, 0.1, 0.3)[(n // 2) % 3], lq == lk)
            for n, (lq, lk) in enumerate((lq, lk) for lq in T5_LQ for lk in T5_LK)]


def _t5_inputs(B, Lq, Lk, H, dh, with_bias, with_pad, seed):
    """K and V are the two column halves of one [B, Lk, 2D] tensor, as _T5AttnFn passes them.  Padding: every key of batch row 0,
    all but the last key of row 1, the tail of row 2."""
    from genrec_b200.t5_attention import relative_position_buckets
    g = torch.Generator().manual_seed(seed)
    D = H * dh
    Q = (2 * torch.randn(B, Lq, D, generator=g)).bfloat16().to(DEV)
    KV = torch.randn(B, Lk, 2 * D, generator=g).bfloat16().to(DEV)
    dO = torch.randn(B, Lq, D, generator=g).bfloat16().to(DEV)
    bias = (1.5 * torch.randn(H, 32, generator=g)).to(DEV) if with_bias else None
    bucket = relative_position_buckets(Lq, Lk).to(DEV) if with_bias else None
    pad = None
    if with_pad:
        pad = torch.zeros(B, Lk, dtype=torch.uint8)
        pad[0] = 1
        pad[1, :-1] = 1
        pad[2, Lk - Lk // 3:] = 1
        pad = pad.to(DEV)
    return Q, KV[..., :D], KV[..., D:], dO, bias, bucket, pad


def _t5_check(tag, B, Lq, Lk, H, dh, with_bias, with_pad, p, causal, seed=5, site=3):
    from genrec_b200 import t5_attention as t5
    Q, K, V, dO, bias, bucket, pad = _t5_inputs(B, Lq, Lk, H, dh, with_bias, with_pad, Lq * 1000 + Lk + dh)
    scale = 1 / math.sqrt(dh)
    out, lse = t5.attention_core_fwd(Q, K, V, H, bias, bucket, pad, causal, scale, p, seed, site)
    dq, dk, dv, dbias = t5.attention_core_bwd(Q, K, V, H, bias, bucket, pad, causal, scale, out, lse, dO, p, seed, site)
    ref = ar.t5_reference(Q, K, V, H, bias, bucket, pad, causal, scale, dO, out, p, seed, site)
    got = {"out": out, "dq": dq, "dk": dk, "dv": dv}
    if bias is not None:
        got["dbias"] = dbias
    err = ar.errors(got, ref, ("out", "dq", "dk", "dv", "dbias"))
    _report(tag, err)
    assert not ar.violations(err, "t5"), ar.fmt(err)
    assert not ar.t5_exact(got, ref, pad)
    # the saved softmax statistics: row max and sum (a fully padded row: max -1e9, sum = its number of visible keys)
    m, l = lse[..., 0].double(), lse[..., 1].double()
    assert ((m - ref["m"]).abs() <= 1e-4 * (1 + ref["m"].abs())).all()
    assert ((l - ref["l"]).abs() <= 1e-4 * ref["l"]).all()
    return ref


@pytest.mark.parametrize("Lq,Lk,dh,with_bias,with_pad,p,causal", T5_CASES)
def test_t5_core_vs_fp64(Lq, Lk, dh, with_bias, with_pad, p, causal):
    _t5_check(f"t5 Lq={Lq} Lk={Lk} dh={dh} bias={with_bias} pad={with_pad} p={p} causal={causal}", 3, Lq, Lk, 2, dh, with_bias,
              with_pad, p, causal)


def test_t5_fully_padded_row_is_uniform():
    """A row whose keys are all padded: the reference's -1e9 fill gives a uniform softmax, so O is the mean of V."""
    ref = _t5_check("t5 padded rows", 3, 33, 65, 2, 32, True, True, 0.0, False)
    assert torch.allclose(ref["out"][0], ref["out"][0, :1].expand_as(ref["out"][0]))


def test_t5_generate_cross_attention_shape():
    """generate's cross-attention (tiger.py): D = 384, H = 6, each user's K = 10 beams x (s + 1) = 4 queries against 61 memory rows
    with a tail padding of 20, no bias."""
    from genrec_b200 import t5_attention as t5
    B, R, S, Lk, D, H = 8, 10, 4, 61, 384, 6
    g = torch.Generator().manual_seed(61)
    Q = torch.randn(B, R * S, D, generator=g).bfloat16().to(DEV)
    KV = torch.randn(B, Lk, 2 * D, generator=g).bfloat16().to(DEV)
    dO = torch.randn(B, R * S, D, generator=g).bfloat16().to(DEV)
    pad = torch.zeros(B, Lk, dtype=torch.uint8)
    pad[:, Lk - 20:] = 1
    pad = pad.to(DEV)
    K, V = KV[..., :D], KV[..., D:]
    scale = 1 / math.sqrt(D // H)
    out, lse = t5.attention_core_fwd(Q, K, V, H, None, None, pad, False, scale)
    dq, dk, dv, _ = t5.attention_core_bwd(Q, K, V, H, None, None, pad, False, scale, out, lse, dO)
    ref = ar.t5_reference(Q, K, V, H, None, None, pad, False, scale, dO, out)
    err = ar.errors({"out": out, "dq": dq, "dk": dk, "dv": dv}, ref, ("out", "dq", "dk", "dv"))
    _report("t5 generate cross-attention", err)
    assert not ar.violations(err, "t5"), ar.fmt(err)
    assert not bool(dk[pad.bool()].any()) and not bool(dv[pad.bool()].any())


@pytest.mark.parametrize("B,L", [(256, 61), (16, 130)])
def test_t5_backward_is_reproducible(B, L):
    """The T5 core backward, run twice, gives the same bits in dQ, dK, dV and dbias: the bias bins are summed in a fixed order and,
    from three query tiles on, dK / dV from per-tile partials."""
    from genrec_b200 import t5_attention as t5
    H, dh = 6, 64
    Q, K, V, dO, bias, bucket, pad = _t5_inputs(B, L, L, H, dh, True, True, B + L)
    scale = 1 / math.sqrt(dh)
    out, lse = t5.attention_core_fwd(Q, K, V, H, bias, bucket, pad, False, scale, 0.1, 9, 4)
    first = t5.attention_core_bwd(Q, K, V, H, bias, bucket, pad, False, scale, out, lse, dO, 0.1, 9, 4)
    second = t5.attention_core_bwd(Q, K, V, H, bias, bucket, pad, False, scale, out, lse, dO, 0.1, 9, 4)
    for name, a, b in zip(("dq", "dk", "dv", "dbias"), first, second):
        assert torch.equal(a, b), name


def test_tiger_training_step_is_reproducible(golden):
    """Forward and backward of tiger_small.pt's model, run twice from the same seeds and dropout sites: every .grad is the same bits."""
    from genrec_b200 import t5_attention, tiger
    from genrec_b200.tiger import Tiger
    from tests import tiger_params as tp
    g = golden("tiger_small.pt")
    m = Tiger(**g["cfg"])
    m.load_state_dict(tp.tiger_params(g["shapes"], g["param_seed"]), strict=True)
    m = m.to(DEV).train()
    batch = {k: v.to(DEV) for k, v in tp.batch(g["cfg"], g["B"], g["n_items"], g["batch_seed"]).items()}
    sites = (t5_attention._CALLS["n"], tiger._SITES["n"])

    def run():
        t5_attention._CALLS["n"], tiger._SITES["n"] = sites
        torch.manual_seed(123)
        m.zero_grad(set_to_none=True)
        m(**batch).loss.backward()
        return {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}

    first, second = run(), run()
    assert len(first) > 10
    for n in first:
        assert torch.equal(first[n], second[n]), n


# ------------------------------------------------------------------------------------------------ d-activation GEMM
@pytest.mark.parametrize("T", [1, 77, 129, 25600])
@pytest.mark.parametrize("N,K", [(776, 136), (1024, 384), (384, 1024)])
@pytest.mark.parametrize("act,p", [(1, 0.0), (2, 0.2), (1, 0.2), (2, 0.0)])
def test_linear_dact_bwd_vs_fp64(T, N, K, act, p):
    """g = bf16(mask scale (dy W) act'(z)) against fp64 on the same bf16 operands: within half a bf16 ulp plus the fp32 accumulation
    of the N-term products (and the approximate sigmoid of silu')."""
    import genrec_b200.functional as Fn
    gen = torch.Generator().manual_seed(T + N + K + act)
    dy = torch.randn(T, N, generator=gen).bfloat16().to(DEV)
    w = (0.1 * torch.randn(N, K, generator=gen)).bfloat16().to(DEV)
    z = (2 * torch.randn(T, K, generator=gen)).bfloat16().to(DEV)
    seed, site = 4242, 9
    got = Fn.linear_dact_bwd(dy, w, z, act, p=p, seed=seed, site=site).double()
    acc = dy.double() @ w.double()
    mag = dy.double().abs() @ w.double().abs()
    zz = z.double()
    if act == 1:
        s = torch.sigmoid(zz)
        d = s * (1 + zz * (1 - s))
    else:
        d = (zz > 0).double()
    _, sc = ar.keep_scale(p)
    keep = torch.from_numpy(~ar.drop_mask(range(T), K, p, seed, site)).to(DEV).double() * sc
    ref = acc * d * keep
    # silu' = s (1 + z (1 - s)) from the approximate sigmoid cancels near its zero: its error is bounded absolutely
    allow = ar.U * ref.abs() + (N * 2.0 ** -23 * mag * d.abs() + 2.0 ** -18 * acc.abs() * (1 + zz.abs())) * keep
    r = ((got - ref).abs() / allow.clamp_min(1e-30)).max().item()
    print(f"dact T={T} N={N} K={K} act={act} p={p}: worst {r:.3f}")
    assert r <= 1.0, r                      # a bound, not a measured tolerance: measured 0.95 (T = 25600, N = 384, K = 1024, act = 1)
    assert not bool(got[keep == 0].any())
