"""The checks of tests/attention_reference.py catch what they claim to, without a GPU.

An fp32 model of each attention kernel - SASRec's online softmax over 64-key tiles with bf16 packing of P and dS where
csrc/attn_sasrec.cuh packs them, and the fp32 T5 core of csrc/attn_t5.cuh - must pass every check at the tolerances the GPU tests
use; each mutant plants one plausible defect of a rewritten kernel and must fail them."""
import math

import pytest
import torch

from tests import attention_reference as ar

SAS_DEFECTS = ["causal off by one", "key padding ignored", "padded query row not zeroed", "dropout not in dA", "dropout row/col swapped",
               "missing keep scale", "Dsum from dropped P", "dS missing scale", "lse from dropped P"]
T5_DEFECTS = ["causal off by one", "key padding ignored", "-inf fill", "keys past Lk in softmax", "dropout not in dA",
              "dropout row/col swapped", "missing keep scale", "Dsum from dropped P", "dS missing scale", "bucket at i - j",
              "dbias includes padded cells", "lse from dropped P"]


def _bf(x):
    return x.bfloat16().float()


def _heads(x, H):
    B, L, D = x.shape
    return x.float().reshape(B, L, H, D // H).transpose(1, 2)


def _merge(x):
    B, H, L, dh = x.shape
    return x.transpose(1, 2).reshape(B, L, H * dh)


def _keep(B, H, Lq, Lk, p, seed, site, defects):
    keep = ar.attn_keep(B, H, Lq, Lk, p, seed, site).float()
    if "dropout row/col swapped" in defects:
        keep = ar.attn_keep(B, H, Lk, Lq, p, seed, site).float().transpose(-1, -2)
    if "missing keep scale" in defects:
        keep = (keep > 0).float()
    return keep


# ------------------------------------------------------------------------------------------------ fp32 models of the kernels
def sas_model(Q, K, V, pad, H, dO, p, seed, layer, defects=()):
    B, L, D = Q.shape
    dh = D // H
    scale = ar.f32(1.0 / math.sqrt(dh))
    q, k, v, do = _heads(Q, H), _heads(K, H), _heads(V, H), _heads(dO, H)
    padb = pad.bool()
    i = torch.arange(L)[:, None]
    j = torch.arange(L)[None, :]
    causal = (j < i) if "causal off by one" in defects else (j <= i)
    valid = causal[None, None].expand(B, H, L, L)
    if "key padding ignored" not in defects:
        valid = valid & ~padb[:, None, None, :]
    if "padded query row not zeroed" not in defects:
        valid = valid & ~padb[:, None, :, None]
    keep = _keep(B, H, L, L, p, seed, ar.sas_site(layer), defects)
    S = (q @ k.transpose(-1, -2)) * scale
    S = S.masked_fill(~valid, float("-inf"))
    m = torch.full((B, H, L, 1), float("-inf"))
    l = torch.zeros(B, H, L, 1)
    o = torch.zeros(B, H, L, dh)
    for k0 in range(0, L, 64):
        s = S[..., k0:k0 + 64]
        nm = torch.maximum(m, s.amax(-1, keepdim=True))
        al = torch.where(nm == float("-inf"), torch.ones_like(nm), torch.exp(m - nm))
        pt = torch.where(s == float("-inf"), torch.zeros_like(s), torch.exp(s - nm))
        pd = pt * keep[..., k0:k0 + 64]
        l = l * al + (pd if "lse from dropped P" in defects else pt).sum(-1, keepdim=True)
        o = o * al + _bf(pd) @ v[..., k0:k0 + 64, :]
        m = nm
    out = _bf(torch.where(l > 0, o / l, torch.zeros_like(o)))
    lse = torch.where(l > 0, m + torch.log(l), torch.zeros_like(l))
    # backward
    P = torch.where(valid, torch.exp(S - lse), torch.zeros_like(S))
    dA = do @ v.transpose(-1, -2)
    dAd = dA if "dropout not in dA" in defects else keep * dA
    Dsum = (do * out).sum(-1, keepdim=True)
    if "Dsum from dropped P" in defects:
        Dsum = (P * keep * dAd).sum(-1, keepdim=True)
    ds = torch.where(valid, P * (dAd - Dsum), torch.zeros_like(P))
    if "dS missing scale" not in defects:
        ds = ds * scale
    ds = _bf(ds)
    got = {"out": _merge(out), "lse": lse[..., 0], "dq": _merge(_bf(ds @ k)), "dk": _merge(_bf(ds.transpose(-1, -2) @ q)),
           "dv": _merge(_bf(_bf(P * keep).transpose(-1, -2) @ do))}
    return got


def t5_model(Q, K, V, H, bias, bucket, key_pad, causal, scale, dO, p, seed, site, defects=()):
    B, Lq, D = Q.shape
    Lk = K.shape[1]
    dh = D // H
    scale = ar.f32(scale)
    q, k, v, do = _heads(Q, H), _heads(K, H), _heads(V, H), _heads(dO, H)
    Lx = Lk
    if "keys past Lk in softmax" in defects:                  # the zero-filled rows of the last 64-key tile take part
        Lx = (Lk + 63) // 64 * 64
        k = torch.cat([k, torch.zeros(B, H, Lx - Lk, dh)], 2)
        v = torch.cat([v, torch.zeros(B, H, Lx - Lk, dh)], 2)
    i = torch.arange(Lq)[:, None]
    j = torch.arange(Lx)[None, :]
    S = (q @ k.transpose(-1, -2)) * scale
    if bias is not None:
        delta = (i - j) if "bucket at i - j" in defects else (j - i)
        idx = bucket.long()[(delta + Lq - 1).clamp(0, Lq + Lk - 2)]
        S = S + torch.where(j < Lk, bias[:, idx], torch.zeros(()))[None]
    kp = torch.zeros(B, 1, 1, Lx, dtype=torch.bool)
    if key_pad is not None and "key padding ignored" not in defects:
        kp[..., :Lk] = key_pad.bool()[:, None, None, :]
        S = torch.where(kp, torch.full_like(S, float("-inf") if "-inf fill" in defects else -1e9), S)
    excl = torch.zeros(Lq, Lx, dtype=torch.bool)
    if causal:
        excl = (j > i + 1) if "causal off by one" in defects else (j > i)
    S = S.masked_fill(excl[None, None], float("-inf"))
    m = S.amax(-1, keepdim=True)
    dead = m == float("-inf")
    E = torch.where(dead, torch.zeros_like(S), torch.exp(S - torch.where(dead, torch.zeros_like(m), m)))
    keep = _keep(B, H, Lq, Lx, p, seed, site, defects)
    l = (E * keep if "lse from dropped P" in defects else E).sum(-1, keepdim=True)
    inv = torch.where(l > 0, 1 / l, torch.zeros_like(l))
    P = E * inv
    out = _bf(P * keep @ v)
    dA = do @ v.transpose(-1, -2)
    dAd = dA if "dropout not in dA" in defects else keep * dA
    Dsum = (do * out).sum(-1, keepdim=True)
    if "Dsum from dropped P" in defects:
        Dsum = (P * keep * dAd).sum(-1, keepdim=True)
    ds = P * (dAd - Dsum)
    ds_db = torch.where(excl[None, None], torch.zeros_like(ds), ds)
    ds = torch.where(kp | excl[None, None], torch.zeros_like(ds), ds)
    dss = ds if "dS missing scale" in defects else ds * scale
    got = {"out": _merge(out), "dq": _merge(_bf(dss @ k)), "dk": _merge(dss.transpose(-1, -2) @ q)[:, :Lk],
           "dv": _merge((P * keep).transpose(-1, -2) @ do)[:, :Lk]}
    if bias is not None:
        src = ds_db if "dbias includes padded cells" in defects else ds
        delta = (i - j) if "bucket at i - j" in defects else (j - i)
        idx = bucket.long()[(delta + Lq - 1).clamp(0, Lq + Lk - 2)][:, :Lk]
        got["dbias"] = torch.zeros(B, H, bias.shape[1]).scatter_add_(2, idx.expand(B, H, Lq, Lk).reshape(B, H, -1),
                                                                      src[..., :Lk].reshape(B, H, -1)).sum(0)
    return got


# ------------------------------------------------------------------------------------------------ cases
def sas_case(B, L, H, dh, seed, spread=1.0):
    g = torch.Generator().manual_seed(seed)
    D = H * dh
    Q = (spread * torch.randn(B, L, D, generator=g)).bfloat16()
    K = torch.randn(B, L, D, generator=g).bfloat16()
    V, dO = torch.randn(B, L, D, generator=g).bfloat16(), torch.randn(B, L, D, generator=g).bfloat16()
    pad = torch.zeros(B, L, dtype=torch.uint8)
    pad[0, :5] = 1                                       # left padding
    if B > 1:
        pad[1, L // 3: L // 3 + 7] = 1                   # a hole in the middle
        pad[1, L - 3:] = 1                               # tail padding
    if B > 2:
        pad[2] = 1                                       # a fully padded sequence
    return Q, K, V, dO, pad


def t5_case(B, Lq, Lk, H, dh, seed, bias=True, spread=1.0):
    from genrec_b200.t5_attention import relative_position_buckets
    g = torch.Generator().manual_seed(seed)
    D = H * dh
    Q = (spread * torch.randn(B, Lq, D, generator=g)).bfloat16()
    KV = torch.randn(B, Lk, 2 * D, generator=g).bfloat16()
    dO = torch.randn(B, Lq, D, generator=g).bfloat16()
    b = (0.7 * torch.randn(H, 32, generator=g)) if bias else None
    bk = relative_position_buckets(Lq, Lk) if bias else None
    pad = torch.zeros(B, Lk, dtype=torch.uint8)
    pad[0] = 1                                           # every key padded: a uniform softmax
    if B > 1:
        pad[1, Lk - 7:] = 1
    if B > 2:
        pad[2, :-1] = 1                                  # only the last key valid
    return Q, KV[..., :D], KV[..., D:], dO, b, bk, pad


def _sas_errors(case, H, p, defects=()):
    Q, K, V, dO, pad = case
    got = sas_model(Q, K, V, pad, H, dO, p, 99, 1, defects)
    ref = ar.sasrec_reference(Q, K, V, pad, H, dO, got["out"].bfloat16(), p, 99, 1)
    err = ar.errors(got, ref, ("out", "dq", "dk", "dv"))
    return ar.violations(err, "sas") + ar.sasrec_exact(got, ref), err


def _t5_errors(case, H, causal, p, defects=()):
    Q, K, V, dO, b, bk, pad = case
    scale = 1 / math.sqrt(Q.shape[-1] // H)
    got = t5_model(Q, K, V, H, b, bk, pad, causal, scale, dO, p, 5, 17, defects)
    ref = ar.t5_reference(Q, K, V, H, b, bk, pad, causal, scale, dO, got["out"].bfloat16(), p, 5, 17)
    err = ar.errors(got, ref, ("out", "dq", "dk", "dv", "dbias"))
    return ar.violations(err, "t5") + ar.t5_exact(got, ref, pad), err


SAS_CASES = [(dict(B=3, L=130, H=2, dh=32, seed=1, spread=3.0), 0.0), (dict(B=3, L=130, H=2, dh=32, seed=2, spread=3.0), 0.2),
             (dict(B=2, L=65, H=1, dh=64, seed=3), 0.5)]
T5_CASES = [(dict(B=3, Lq=40, Lk=40, H=2, dh=32, seed=4), True, 0.0), (dict(B=3, Lq=70, Lk=70, H=2, dh=32, seed=5, spread=2.0), False, 0.2),
            (dict(B=3, Lq=5, Lk=61, H=2, dh=64, seed=6, bias=False, spread=0.3), False, 0.1)]


def test_models_pass():
    for kw, p in SAS_CASES:
        bad, err = _sas_errors(sas_case(**kw), kw["H"], p)
        assert not bad, (kw, p, bad, ar.fmt(err))
    for kw, causal, p in T5_CASES:
        bad, err = _t5_errors(t5_case(**kw), kw["H"], causal, p)
        assert not bad, (kw, p, bad, ar.fmt(err))


@pytest.mark.parametrize("defect", SAS_DEFECTS)
def test_sasrec_mutant_fails(defect):
    fails = [_sas_errors(sas_case(**kw), kw["H"], p, (defect,))[0] for kw, p in SAS_CASES]
    assert any(fails), defect


@pytest.mark.parametrize("defect", T5_DEFECTS)
def test_t5_mutant_fails(defect):
    fails = [_t5_errors(t5_case(**kw), kw["H"], causal, p, (defect,))[0] for kw, causal, p in T5_CASES]
    assert any(fails), defect


def _np_drop_mask(T, D, p, seed, site):
    """numpy restatement of genrec_b200/csrc/common.cuh Dropout (row keys + pair hash); True = dropped."""
    import numpy as np
    u = np.uint32
    k0 = u((seed & 0xffffffff) ^ ((site * 0x9E3779B1) & 0xffffffff))
    k1 = u(((seed >> 32) + 0x7F4A7C15) & 0xffffffff)
    row = np.arange(T, dtype=np.uint32)[:, None]
    cp = np.arange(D // 2, dtype=np.uint32)[None, :]
    with np.errstate(over="ignore"):
        ka = (row ^ k1) * u(0x9E3779B1)
        ka = ka ^ (ka >> u(16))
        b = ka * u(0x846CA68B)
        kb = k0 ^ (b ^ (b >> u(15)))
        x = (cp ^ kb) * u(0x7FEB352D)
        x = x ^ (x >> u(15))
        x = (x ^ ka) * u(0x846CA68B)
        x = x ^ (x >> u(16))
    t = u(int(p * 65536.0 + 0.5))
    m = np.empty((T, D), dtype=bool)
    m[:, 0::2] = (x & u(0xffff)) < t
    m[:, 1::2] = (x >> u(16)) < t
    return m


def test_drop_mask_matches_the_paired_column_form():
    """drop_mask on rows 0 .. T - 1 is _np_drop_mask's [T, D] mask, restated in the paired-column form of csrc/common.cuh."""
    for T, D, p, seed, site in [(77, 136, 0.2, 1234567, 6), (5, 9, 0.5, (3 << 40) + 5, 11)]:
        m = ar.drop_mask(range(T), D, p, seed, site)
        if D % 2 == 0:
            assert (m == _np_drop_mask(T, D, p, seed, site)).all()
        assert abs(m.mean() - p) < 0.1
    assert not ar.drop_mask(range(4), 8, 0.0, 1, 1).any()
