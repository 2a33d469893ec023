"""fp64 references of the SASRec attention core (csrc/attn_sasrec.cuh) and the T5 attention core (csrc/attn_t5.cuh) that know where
the kernels round, the dropout mask they share, and the checks with their tolerances.

Both references take the kernels' own bf16 Q, K, V and dO, and for the backward's Dsum = rowsum(dO * O) the kernel's own bf16 O:
both backward kernels read the rounded O (sas_rowdot, t5_load_row(o, a.out ...)).  Everything else is exact fp64 math.  The
rounding of the kernels is not replayed but bounded per element: each output element gets an allowance built from the magnitudes
of the terms it sums, and the checks divide the error by it.

SASRec rounds on purpose in these places (mma.sync path, fp32 accumulation):
  1. the forward's unnormalised probabilities, after dropout, are packed to bf16 before P V (att_pack_p).  The row sum l is taken
     from the unrounded values, so rounding 1 moves each term of O by at most 2^-8 of |P_ij V_jd|.
  2. the backward's dS (dq and dkdv kernels) and the dropped P (dV) are packed to bf16 before their MMAs: 2^-8 of each term.
  3. O, dQ, dK and dV are stored as bf16, round to nearest even: 2^-8 of the result.
  4. exp is __expf, scores and sums are fp32: a few 2^-24 per term (GAMMA below), and for dS the absolute fp32 error of dA and
     Dsum, which cancel against each other in dA - Dsum.
The T5 core is fp32 CUDA-core throughout: only O and dQ are rounded to bf16 (3); dK, dV and dbias are fp32, so their allowance is
the fp32 accumulation bound alone.

Dropout: `drop_mask` restates Dropout::apply of csrc/common.cuh bit for bit.  SASRec uses row key (b H + h) L + i and column j at
site 8 layer + 3; T5 uses row key (b H + h) Lq + i and column j at the caller's site.
"""
import math

import numpy as np
import torch

U = 2.0 ** -8                     # bf16 round-to-nearest-even, relative: half an ulp of an 8-bit significand
GAMMA_SLACK = 2.0 ** -17          # __expf / exp_accurate and the fp32 score error, relative to each probability

# ---- tolerances.  `worst` = max over elements of |got - ref| / allowance, `frob` = |got - ref|_F / |allowance|_F.  Each is ~3x the
#      largest value measured over every case of tests/test_attention_exact_gpu.py on an H100 80GB HBM3 (700 W power limit); the
#      measured value is quoted beside it.  tests/test_attention_reference_cpu.py checks that every mutant of the kernels it models is
#      rejected at these values.
TOL = {
    # SASRec, every output: measured worst 0.95 (dv, L = 200, d/H = 64, p = 0.2), frob 0.30 (dk, L = 17, d/H = 32, H = 4, p = 0.5)
    "sas worst": 2.8,
    "sas frob": 0.9,
    # T5 bf16 outputs (out, dq): measured worst 0.99 (out, Lq = 64, Lk = 4), frob 0.50 (out, Lq = 130, Lk = 61)
    "t5 bf16 worst": 3.0,
    "t5 bf16 frob": 1.5,
    # T5 fp32 outputs (dk, dv, dbias): measured worst 0.106 (dv, Lq = 1, Lk = 65, p = 0.3), frob 0.0122 (dv, Lq = 4, Lk = 200).  The
    # largest errors sit in dV at one to four query rows, where the fp32 score error moves P by more than GAMMA_SLACK
    "t5 fp32 worst": 0.32,
    "t5 fp32 frob": 0.037,
}
T5_BF16 = ("out", "dq")


# ------------------------------------------------------------------------------------------------ dropout
def keep_scale(p):
    """(threshold, keep scale) of make_dropout: thresh = round(p 2^16), scale = 2^16 / (2^16 - thresh) in fp32."""
    if p <= 0:
        return 0, 1.0
    t = min(int(p * 65536.0 + 0.5), 65536)
    return t, float(np.float32(65536.0) / np.float32(65536 - t)) if t < 65536 else 0.0


def drop_mask(rows, ncols, p, seed, site):
    """Dropout::apply's mask: rows (array of uint32 row keys) x columns 0 .. ncols - 1, True = dropped.  One pair hash serves
    columns 2c and 2c + 1, the low 16 bits for the even column and the high 16 for the odd one."""
    u = np.uint32
    rows = np.asarray(rows, dtype=np.uint64).astype(np.uint32)[:, None]
    thresh, _ = keep_scale(p)
    if thresh == 0:
        return np.zeros((rows.shape[0], ncols), dtype=bool)
    k0 = u((seed & 0xffffffff) ^ ((site * 0x9E3779B1) & 0xffffffff))
    k1 = u(((seed >> 32) + 0x7F4A7C15) & 0xffffffff)
    cp = np.arange((ncols + 1) // 2, dtype=np.uint32)[None, :]
    with np.errstate(over="ignore"):
        ka = (rows ^ k1) * u(0x9E3779B1)
        ka = ka ^ (ka >> u(16))
        b = ka * u(0x846CA68B)
        kb = k0 ^ (b ^ (b >> u(15)))
        x = (cp ^ kb) * u(0x7FEB352D)
        x = x ^ (x >> u(15))
        x = (x ^ ka) * u(0x846CA68B)
        x = x ^ (x >> u(16))
    m = np.empty((rows.shape[0], 2 * cp.shape[1]), dtype=bool)
    m[:, 0::2] = (x & u(0xffff)) < u(thresh)
    m[:, 1::2] = (x >> u(16)) < u(thresh)
    return m[:, :ncols]


def attn_keep(B, H, Lq, Lk, p, seed, site, device="cpu"):
    """[B, H, Lq, Lk] fp64 keep-scale matrix (0 where dropped) of an attention core, row key (b H + h) Lq + i, column j."""
    drop = drop_mask(np.arange(B * H * Lq), Lk, p, seed, site)
    _, s = keep_scale(p)
    return torch.from_numpy(np.where(drop, 0.0, s)).view(B, H, Lq, Lk).to(device)


def sas_site(layer):
    return 8 * layer + 3


# ------------------------------------------------------------------------------------------------ reference
def _heads(x, H):
    B, L, D = x.shape
    return x.double().reshape(B, L, H, D // H).transpose(1, 2)


def _merge(x):
    B, H, L, dh = x.shape
    return x.transpose(1, 2).reshape(B, L, H * dh)


def f32(x):
    return float(np.float32(x))


def _core(q, k, v, S, valid, diff, keep, do, o, scale, pack, gamma, gamma_red):
    """Shared fp64 softmax-attention forward / backward with allowances.  S [B, H, Lq, Lk] scores (fp64), valid = cells that take
    part in the softmax, diff = cells whose score depends on q, k (and bias), keep = dropout keep-scale, pack = U where the kernel
    packs P / dS to bf16 (SASRec) else 0."""
    S = S.masked_fill(~valid, float("-inf"))
    m = S.amax(-1, keepdim=True)
    live = valid.any(-1, keepdim=True)
    E = torch.where(valid, torch.exp(S - torch.where(live, m, torch.zeros_like(m))), torch.zeros_like(S))
    l = E.sum(-1, keepdim=True)
    P = torch.where(live, E / l.clamp_min(1e-300), torch.zeros_like(E))
    Pd = P * keep
    r = {"P": P, "keep": keep, "m": m[..., 0], "l": l[..., 0], "live": live[..., 0]}
    r["out"] = Pd @ v
    r["a_out"] = U * r["out"].abs() + (pack + gamma) * (Pd @ v.abs())
    if do is None:
        return r
    dA = do @ v.transpose(-1, -2)
    Dsum = (do * o).sum(-1, keepdim=True)
    ds = torch.where(valid & diff, P * (keep * dA - Dsum), torch.zeros_like(P))
    # dA and Dsum are fp32 dot products of dh terms: their absolute errors enter dS through P (dA - Dsum) undamped by cancellation
    dh = q.shape[-1]
    err_in = dh * 2.0 ** -23 * (keep * (do.abs() @ v.abs().transpose(-1, -2)) + (do.abs() * o.abs()).sum(-1, keepdim=True))
    a_ds = torch.where(valid & diff, (pack + gamma) * ds.abs() + P * err_in, torch.zeros_like(P))
    r["ds"], r["a_ds"] = ds, a_ds
    r["dq"] = scale * (ds @ k)
    r["a_dq"] = U * r["dq"].abs() + scale * (a_ds @ k.abs() + gamma_red * (ds.abs() @ k.abs()))
    r["dk"] = scale * (ds.transpose(-1, -2) @ q)
    r["dv"] = Pd.transpose(-1, -2) @ do
    return r


def sasrec_reference(Q, K, V, pad, H, dO=None, O=None, p=0.0, seed=0, layer=0):
    """Q, K, V, dO, O bf16 [B, L, D] (O: the kernel's forward output), pad [B, L] 1 = padding.  -> dict of [B, L, D] fp64 tensors
    "out", "dq", "dk", "dv" with allowances "a_*", "lse" [B, H, L] (0 where a row has no valid key), the masks "qpad" [B, L] and
    "drop" [B, H, L, L] (True = dropped)."""
    B, L, D = Q.shape
    dh = D // H
    scale = f32(1.0 / math.sqrt(dh))
    q, k, v = _heads(Q, H), _heads(K, H), _heads(V, H)
    padb = pad.bool().to(Q.device)
    i = torch.arange(L, device=Q.device)[:, None]
    j = torch.arange(L, device=Q.device)[None, :]
    valid = ((j <= i)[None, None] & ~padb[:, None, None, :] & ~padb[:, None, :, None]).expand(B, H, L, L)
    keep = attn_keep(B, H, L, L, p, seed, sas_site(layer), Q.device)
    S = (q @ k.transpose(-1, -2)) * scale
    gamma = GAMMA_SLACK + (L + dh) * 2.0 ** -23
    do = _heads(dO, H) if dO is not None else None
    o = _heads(O, H) if O is not None else None
    r = _core(q, k, v, S, valid, valid, keep, do, o, scale, U, gamma, gamma)
    out = {"out": _merge(r["out"]), "a_out": _merge(r["a_out"]), "qpad": padb, "drop": keep == 0,
           "lse": torch.where(r["live"], r["m"] + torch.log(r["l"].clamp_min(1e-300)), torch.zeros_like(r["m"])), "valid": valid}
    if dO is not None:
        a_dk = U * r["dk"].abs() + scale * (r["a_ds"].transpose(-1, -2) @ q.abs() + gamma * (r["ds"].abs().transpose(-1, -2) @ q.abs()))
        Pd = r["P"] * keep
        a_dv = U * r["dv"].abs() + (U + gamma) * (Pd.transpose(-1, -2) @ do.abs())
        out.update(dq=_merge(r["dq"]), a_dq=_merge(r["a_dq"]), dk=_merge(r["dk"]), a_dk=_merge(a_dk), dv=_merge(r["dv"]), a_dv=_merge(a_dv))
    return out


def t5_reference(Q, K, V, H, bias, bucket, key_pad, causal, scale, dO=None, O=None, p=0.0, seed=0, site=0):
    """The T5 core as attention_core_fwd / attention_core_bwd compute it.  Q [B, Lq, D], K, V [B, Lk, D] bf16 (views allowed),
    bias [H, nb] fp32 or None with bucket [Lq + Lk - 1] int32, key_pad [B, Lk] or None.  -> "out", "dq" [B, Lq, D], "dk", "dv"
    [B, Lk, D], "dbias" [H, nb] fp64 with allowances "a_*", "m" / "l" [B, H, Lq] (the softmax statistics the kernel saves)."""
    B, Lq, D = Q.shape
    Lk = K.shape[1]
    dh = D // H
    dev = Q.device
    scale = f32(scale)
    q, k, v = _heads(Q, H), _heads(K, H), _heads(V, H)
    S = (q @ k.transpose(-1, -2)) * scale
    i = torch.arange(Lq, device=dev)[:, None]
    j = torch.arange(Lk, device=dev)[None, :]
    if bias is not None:
        idx = bucket.to(dev).long()[(j - i) + Lq - 1]
        S = S + bias.to(dev).double()[:, idx][None]
    diff = torch.ones(B, 1, 1, Lk, dtype=torch.bool, device=dev)
    if key_pad is not None:
        kp = key_pad.to(dev).bool()[:, None, None, :]
        S = torch.where(kp, torch.full_like(S, -1e9), S)
        diff = ~kp
    valid = ((j <= i) if causal else torch.ones(Lq, Lk, dtype=torch.bool, device=dev))[None, None].expand(B, H, Lq, Lk)
    diff = diff.expand(B, H, Lq, Lk)
    keep = attn_keep(B, H, Lq, Lk, p, seed, site, dev)
    gamma = GAMMA_SLACK + (Lk + dh) * 2.0 ** -23
    do = _heads(dO, H) if dO is not None else None
    o = _heads(O, H) if O is not None else None
    r = _core(q, k, v, S, valid, diff, keep, do, o, scale, 0.0, gamma, gamma)
    out = {"out": _merge(r["out"]), "a_out": _merge(r["a_out"]), "m": r["m"], "l": r["l"], "drop": keep == 0}
    if dO is None:
        return out
    # dK / dV: fp32 sums over the Lq rows, then over the query tiles
    gq = GAMMA_SLACK + (Lq + dh) * 2.0 ** -23
    a_dk = scale * (r["a_ds"].transpose(-1, -2) @ q.abs() + gq * (r["ds"].abs().transpose(-1, -2) @ q.abs()))
    Pd = r["P"] * keep
    a_dv = gq * (Pd.transpose(-1, -2) @ do.abs())
    out.update(dq=_merge(r["dq"]), a_dq=_merge(r["a_dq"]), dk=_merge(r["dk"]), a_dk=_merge(a_dk), dv=_merge(r["dv"]), a_dv=_merge(a_dv))
    if bias is not None:
        nb = bias.shape[1]
        idx = bucket.to(dev).long()[(j - i) + Lq - 1].expand(B, H, Lq, Lk).reshape(B, H, -1)
        db = torch.zeros(B, H, nb, dtype=torch.float64, device=dev).scatter_add_(2, idx, r["ds"].reshape(B, H, -1)).sum(0)
        # per-CTA bins (rows of a tile, diagonals of a bucket) and the ordered sum over B x query tiles
        depth = 32 + Lq + Lk + B * ((Lq + 31) // 32) // 32 + 8
        mag = r["a_ds"] + depth * 2.0 ** -24 * r["ds"].abs()
        a_db = torch.zeros(B, H, nb, dtype=torch.float64, device=dev).scatter_add_(2, idx, mag.reshape(B, H, -1)).sum(0)
        out.update(dbias=db, a_dbias=a_db)
    return out


# ------------------------------------------------------------------------------------------------ checks
def ratios(got, ref, allow):
    """(worst, frob): max |got - ref| / allow over the elements, and |got - ref|_F / |allow|_F.  NaN or Inf gives inf."""
    d = (got.double().to(ref.device) - ref).abs()
    if not bool(torch.isfinite(d).all()):
        return float("inf"), float("inf")
    a = allow.clamp_min(1e-30)
    worst = (d / a).max().item() if d.numel() else 0.0
    n = allow.norm().item()
    return worst, (d.norm().item() / n if n > 0 else (0.0 if d.norm().item() == 0 else float("inf")))


def errors(got, ref, names):
    """{name: (worst, frob)} for each name present in both `got` and `ref`."""
    return {n: ratios(got[n], ref[n], ref["a_" + n]) for n in names if n in got and n in ref}


def tolerance(kind, name):
    """(worst, frob) tolerance of output `name` of kind "sas" or "t5"."""
    if kind == "t5":
        kind += " bf16" if name in T5_BF16 else " fp32"
    return TOL[kind + " worst"], TOL[kind + " frob"]


def violations(err, kind):
    """Names of the checks the (worst, frob) ratios of err fail at the tolerances of kind ("sas" or "t5")."""
    bad = []
    for n, (w, f) in err.items():
        tw, tf = tolerance(kind, n)
        if not (w <= tw and f <= tf):
            bad.append(f"{n} {w:.3g}/{f:.3g}")
    return bad


def sasrec_exact(got, ref):
    """The assertions SASRec must meet exactly: padded query rows give O = 0 and dQ = 0, padded keys dK = dV = 0, a row without a
    valid key has lse = 0, and the forward's dropout zero pattern is the restated mask (checked where it can be seen: P V with
    V = identity, see tests/test_attention_exact_gpu.py).  -> list of the failures."""
    bad = []
    qp = ref["qpad"].to(got["out"].device)
    if bool((got["out"][qp] != 0).any()):
        bad.append("padded query row has O != 0")
    if "dq" in got:
        if bool((got["dq"][qp] != 0).any()):
            bad.append("padded query row has dQ != 0")
        if bool((got["dk"][qp] != 0).any()) or bool((got["dv"][qp] != 0).any()):
            bad.append("padded key has dK or dV != 0")
    if "lse" in got:
        dead = ~ref["valid"].any(-1).to(got["lse"].device)
        if bool((got["lse"][dead] != 0).any()):
            bad.append("row without a valid key has lse != 0")
    return bad


def t5_exact(got, ref, key_pad):
    """T5: a padded key takes no gradient (dK = dV = 0 there unless its whole row of queries is padded and uniform - dV then gets
    the uniform weight, dK stays 0)."""
    bad = []
    if key_pad is not None and "dk" in got:
        kp = key_pad.bool().to(got["dk"].device)
        if bool((got["dk"][kp] != 0).any()):
            bad.append("padded key has dK != 0")
    return bad


def fmt(err):
    return " ".join(f"{n} {w:.2e}/{f:.2e}" for n, (w, f) in err.items())
