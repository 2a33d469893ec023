"""TEST INFRASTRUCTURE - the HSTU cases the GPU tests and their CPU checks share: the bias-table configurations (bucket rules,
tolerances, the attention-core and layer cases and their fp64 restatements), one block's parameters and its packed run through the
C ABI, the serving models, chunks and pool histories of the cached extend, the headline (cfg2) model with its oracle run, and the
synthetic users of the Recall@10 check."""
import ctypes as C

import torch
import torch.nn.functional as F

from tests import dense_reference as dr
from tests import hstu_block_reference as hr
from tests.exact_check import DEV
from tests.util import budget, relerr


# ---- tolerances (max-norm relative error unless stated)
# Attention core on the same bf16 operands as the fp64 restatement: the kernels round A = silu(S) and the outputs to bf16 (2^-9).
CORE_O_TOL = 8e-3
CORE_DZP_TOL = 1.5e-2
# Bias-table row r:  |got_r - ref_r| <= TABLE_C * sum over the cells of bucket r of |dS_ref|.
# The kernel's dS of a cell is computed in fp32 from exact products of bf16 operands (S = Q.K and dA = dO.V, <= 64 terms each), the
# fp32 bias sum and the fast sigmoid (a few ulp): about 1e-5 of |dS| per cell, more only on the rare cells next to the zero of
# silu'.  The row is then an ordered fp32 sum of at most a few hundred terms per level (lane, CTA, sequence): about 2e-5 of the
# mass.  4e-3 leaves two orders of magnitude of headroom; a bucketing mistake moves whole cells, i.e. O(1) of a row's mass.
TABLE_C = 4e-3
# HSTULayer (bf16 path) against the fp64 oracle: the tolerances of test_hstu_gpu.py::test_layer_vs_oracle_shapes
LAYER_Y_TOL = 2.5e-2
LAYER_DX_TOL = 2.5e-2
LAYER_GRAD_TOL = 4e-2
F32_TOL = 1e-5                 # the fp32-exact forward

MAX_TS_SPAN = (1 << 63) - (1 << 56)   # 9.15e18: the reference's time bucket 63, which starts at |dt| ~ 9.14e18


# ---------------------------------------------------------------------------------------------------- bucket rules
def pos_fixed(delta, nb, md):
    """sign-fixed position bucket of cell (i, j), delta = i - j"""
    from oracle import hstu as oh
    return oh.position_bucket(delta, nb, md)


def pos_reference(delta, nb, md):
    """the reference's: bucket(j - i), clamped at 0 - bucket 0 on the whole causal triangle"""
    from oracle import hstu as oh
    return oh.position_bucket(-delta, nb, md)


def time_bucket(dt, nt):
    from oracle import hstu as oh
    return oh.temporal_bucket(dt, nt)


def patch_oracle(monkeypatch, pos_fn, time_fn=time_bucket) -> None:
    """Make oracle.hstu evaluate its bias tables through pos_fn(i - j, num_buckets, max_distance) and time_fn(ts_i - ts_j, nt)."""
    from oracle import hstu as oh

    def position_bias(table, L, num_buckets=32, max_distance=128):
        pos = torch.arange(L, device=table.device)
        return F.embedding(pos_fn(pos[:, None] - pos[None, :], num_buckets, max_distance), table).permute(2, 0, 1)

    def temporal_bias(table, timestamps):
        diff = timestamps.unsqueeze(2) - timestamps.unsqueeze(1)
        return F.embedding(time_fn(diff, table.shape[0]), table).permute(0, 3, 1, 2)

    monkeypatch.setattr(oh, "position_bias", position_bias)
    monkeypatch.setattr(oh, "temporal_bias", temporal_bias)


def sign_fix(module) -> None:
    """Switch every RelativePositionBias of `module` to the sign-fixed table (the one-line change bucket_of_delta documents)."""
    from genrec_b200.hstu import RelativePositionBias
    for m in module.modules():
        if isinstance(m, RelativePositionBias):
            m._relative_position_bucket = (lambda f: (lambda rel: f(-rel)))(m._relative_position_bucket)
            m._table_cache.clear()
            m._uniform_cache.clear()


# ---------------------------------------------------------------------------------------------------- inputs
def batch(L, seed, num_items=500):
    """ids, ts, pad for B = 4: row 0 has a pad in the middle, row 1 is left padded, row 2 fully padded, row 3 spans > 2^62."""
    g = torch.Generator().manual_seed(seed)
    B = 4
    ids = torch.randint(1, num_items + 1, (B, L), generator=g)
    gaps = torch.randint(1, 3 * 86400, (B, L), generator=g)
    gaps[:, ::5] = torch.randint(0, 50, (B, (L + 4) // 5), generator=g)
    ts = 1_300_000_000 + torch.cumsum(gaps, 1)
    ts[3] = 1_300_000_000 + torch.arange(L) * (2 ** 33)
    if L >= 2:
        ts[3, L - 1] = ts[3, 0] + MAX_TS_SPAN
    ids[0, L // 2] = 0
    ids[1, : L // 3] = 0
    ids[2, :] = 0
    pad = ids == 0
    ts[pad] = 0
    return ids, ts, pad


def randomise(module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in module.named_parameters():
            if "attention_bias" in n:
                p.copy_(0.5 * torch.randn(p.shape, generator=g))
            elif n.endswith("bias"):
                p.copy_(0.1 * torch.randn(p.shape, generator=g))
            elif "norm" in n:
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            else:
                p.copy_(0.08 * torch.randn(p.shape, generator=g))
        for n, p in module.named_parameters():
            if n == "item_embedding.weight":
                p[0].zero_()


# ---------------------------------------------------------------------------------------------------- attention core
# pos: ("ref", npos, md) | ("fix", npos, md) ; time: number of buckets, "notable" (timestamps, no table) or "nots" (no timestamps)
def core_case(L, D, H, pos, time, seed):
    """CPU tensors of one attention-core case: bf16 zp, P = silu(zp) and dO; pad; ts (None for "nots"); the tables."""
    g = torch.Generator().manual_seed(seed)
    _, ts, pad = batch(L, seed)
    zp = (0.7 * torch.randn(4, L, 4 * D, generator=g)).to(torch.bfloat16)
    P = F.silu(zp.float()).to(torch.bfloat16)
    dO = (torch.randn(4, L, D, generator=g) / max(1.0, L ** 0.5)).to(torch.bfloat16)
    wpos = 0.3 * torch.randn(pos[1], H, generator=g)
    wtime = 0.5 * torch.randn(time, H, generator=g) if isinstance(time, int) else None
    return dict(zp=zp, P=P, dO=dO, pad=pad, ts=None if time == "nots" else ts, wpos=wpos, wtime=wtime, H=H, pos=pos, time=time)


def cell_buckets(c, pos_fn=None, time_fn=time_bucket):
    """pb [L, L] position bucket and tb [B, L, L] time bucket (None without a time table) of every cell (i, j)."""
    kind, npos, md = c["pos"]
    pos_fn = pos_fn or (pos_fixed if kind == "fix" else pos_reference)
    L = c["pad"].shape[1]
    ii = torch.arange(L)
    pb = pos_fn(ii[:, None] - ii[None, :], npos, md)
    tb = None
    if c["wtime"] is not None and c["ts"] is not None:
        tb = time_fn(c["ts"].unsqueeze(2) - c["ts"].unsqueeze(1), c["wtime"].shape[0])
    return pb, tb


def core_reference(c, pb, tb):
    """fp64 restatement of hstu.py:244-267 on the kernels' bf16 operands, with a per-cell position bucket pb [L, L] and time bucket
    tb [B, L, L] (or None).  -> dict O, dzp, dpos, dtime, dS [B, H, L, L], valid [B, 1, L, L]."""
    P, zp, dO, H = c["P"], c["zp"], c["dO"], c["H"]
    B, L, D4 = P.shape
    D = D4 // 4
    zp64 = zp.double().requires_grad_(True)
    Pf = F.silu(zp64)
    Pq = Pf + (P.double() - Pf).detach()              # forward operands: the bf16 activations; backward through silu(zp)
    U, V, Q, K = Pq.chunk(4, -1)
    hs = lambda t: t.reshape(B, L, H, D // H).transpose(1, 2)
    wpos = c["wpos"].double().requires_grad_(True)
    S = hs(Q) @ hs(K).transpose(-1, -2) + wpos[pb].permute(2, 0, 1)[None]
    wtime = None
    if tb is not None:
        wtime = c["wtime"].double().requires_grad_(True)
        S = S + wtime[tb].permute(0, 3, 1, 2)
    S.retain_grad()
    ii = torch.arange(L)
    valid = (ii[None, :] <= ii[:, None])[None, None] & ~c["pad"][:, None, None, :]
    A = torch.where(valid, F.silu(S), torch.zeros_like(S))
    O = (A @ hs(V)).transpose(1, 2).reshape(B, L, D)
    O.backward(dO.double())
    return dict(O=O.detach(), dzp=zp64.grad, dpos=wpos.grad, dtime=wtime.grad if wtime is not None else None, dS=S.grad, valid=valid)


def bucket_mass(ref, cells, nrows):
    """(mass [nrows, H] = sum of |dS_ref| over each bucket's valid cells, count [nrows] of valid cells)"""
    dS, valid = ref["dS"], ref["valid"][:, 0]
    B, H = dS.shape[:2]
    idx = cells.expand(B, -1, -1)[valid]
    mass = torch.zeros(nrows, H, dtype=torch.float64)
    for h in range(H):
        mass[:, h].index_add_(0, idx, dS[:, h][valid].abs())
    return mass, torch.bincount(idx, minlength=nrows)


def table_excess(got, want, mass, count) -> float:
    """max over rows of |got_r - want_r| / (TABLE_C * mass_r); a row no cell maps to must be exactly 0 (else inf)."""
    got, want = got.double().cpu(), want.double().cpu()
    if bool((got[count == 0] != 0).any()) or bool((want[count == 0] != 0).any()):
        return float("inf")
    live = count > 0
    diff, m = (got - want).abs()[live], TABLE_C * mass[live]
    if bool(((m == 0) & (diff > 0)).any()):
        return float("inf")
    return float((diff / m.clamp(min=1e-300)).max()) if diff.numel() else 0.0


def core_excess(got, ref, pb, tb, D) -> dict:
    """each checked quantity's error divided by its tolerance (<= 1 passes): O, the V/Q/K columns of dzp, dpos and dtime rows."""
    out = {"O": relerr(got["O"], ref["O"]) / CORE_O_TOL}
    for name, lo in (("dV", D), ("dQ", 2 * D), ("dK", 3 * D)):
        out[name] = relerr(got["dzp"][..., lo:lo + D], ref["dzp"][..., lo:lo + D]) / CORE_DZP_TOL
    npos = ref["dpos"].shape[0]
    out["dpos"] = table_excess(got["dpos"], ref["dpos"], *bucket_mass(ref, pb[None], npos))
    if ref["dtime"] is not None:
        out["dtime"] = table_excess(got["dtime"], ref["dtime"], *bucket_mass(ref, tb, ref["dtime"].shape[0]))
    return out


# (L, D, H, pos, time): every L of the tile edges, head_dim 32 and 64, all four dK/dV instantiations (time table or not x uniform
# or per-bucket positions), npos = 64 with a time table (the dK/dV kernel's largest shared-memory launch) at both head dims
CORE_CASES = [
    (1, 64, 2, ("fix", 8, 12), 20),
    (7, 128, 4, ("fix", 32, 100), 63),
    (64, 128, 2, ("fix", 64, 80), 64),
    (65, 64, 2, ("ref", 32, 128), 20),
    (127, 128, 4, ("ref", 32, 128), 63),
    (200, 128, 2, ("fix", 8, 12), 1),
    (257, 128, 4, ("fix", 64, 80), 20),
    (257, 128, 2, ("ref", 32, 128), 1),
    (200, 128, 4, ("ref", 32, 128), "notable"),
    (130, 128, 2, ("fix", 32, 100), "nots"),
    (64, 128, 4, ("fix", 64, 80), "notable"),
    (65, 128, 2, ("ref", 32, 128), "nots"),
    (127, 128, 2, ("fix", 64, 80), 63),
    (7, 64, 2, ("ref", 32, 128), 64),
    (200, 128, 2, ("fix", 32, 100), 20),
    (257, 64, 2, ("fix", 8, 12), 64),
]


def core_id(case):
    L, D, H, pos, time = case
    return f"L{L}-dh{D // H}-{pos[0]}{pos[1]}md{pos[2]}-t{time}"


# ---------------------------------------------------------------------------------------------------- HSTULayer
# (B = 4, L, D, H, npos, md, ntime): sign-fixed buckets
LAYER_CASES = [(200, 128, 4, 16, 40, 20), (65, 128, 2, 64, 80, 63), (257, 128, 4, 64, 80, 20), (130, 128, 2, 16, 40, 63)]
# the fp32-exact forward
F32_LAYER_CASES = [(130, 128, 4, 16, 40, 20), (200, 128, 2, 64, 80, 64), (65, 64, 2, 32, 100, 20)]


def layer_case(L, D, H, npos, md, ntime, seed):
    from genrec_b200.hstu import HSTULayer
    torch.manual_seed(seed)
    layer = HSTULayer(D, H, 0.0, npos, ntime, md, True)
    randomise(layer, seed)
    _, ts, pad = batch(L, seed)
    g = torch.Generator().manual_seed(seed + 1)
    x = torch.randn(4, L, D, generator=g)
    dy = torch.randn(4, L, D, generator=g)
    return dict(layer=layer, sd={k: v.detach().clone() for k, v in layer.state_dict().items()}, x=x, dy=dy, ts=ts, pad=pad, H=H,
                npos=npos, md=md)


def oracle_layer(c, with_grad=True):
    """fp64 oracle of one block (through whatever bucket rules patch_oracle installed) -> y, dx, {param: grad}"""
    from oracle import hstu as oh
    sd = {k: v.double().requires_grad_(with_grad) for k, v in c["sd"].items()}
    x = c["x"].double().requires_grad_(with_grad)
    y = oh.hstu_layer_forward(x, c["pad"], c["ts"], sd, "", c["H"], True, c["npos"], c["md"])
    if not with_grad:
        return y.detach(), None, None
    y.backward(c["dy"].double())
    return y.detach(), x.grad, {k: v.grad for k, v in sd.items()}


def layer_excess(y, dx, grads, ref) -> dict:
    yr, dxr, gr = ref
    out = {"y": relerr(y, yr) / LAYER_Y_TOL}
    if dx is not None:
        out["dx"] = relerr(dx, dxr) / LAYER_DX_TOL
        for n, g in grads.items():
            out[n] = relerr(g, gr[n]) / LAYER_GRAD_TOL
    return out


# ---------------------------------------------------------------------------------------------------- one block
def _params(D, H, npos, ntime, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s: torch.randn(*s, generator=g)                            # noqa: E731
    wp = 0.08 * r(4 * D, D)
    wp -= wp.mean(1, keepdim=True)          # rows summing to ~0: the +-1000 row offsets of x stay out of the projection
    p = dict(proj_w=wp, proj_b=0.1 * r(4 * D), pos_table=0.3 * r(npos, H), time_table=0.5 * r(max(ntime, 1), H),
             ln1_g=1 + 0.1 * r(D), ln1_b=0.1 * r(D), ffn1_w=0.08 * r(4 * D, D), ffn1_b=0.1 * r(4 * D), ffn2_w=0.08 * r(D, 4 * D),
             ffn2_b=0.1 * r(D), ln2_g=1 + 0.1 * r(D), ln2_b=0.1 * r(D))
    p = {k: v.to(DEV) for k, v in p.items()}
    for k in ("proj_w", "ffn1_w", "ffn2_w"):
        p[k] = p[k].bfloat16()
    return p


def _attn_case(L, D, H, pos, time, seed, ledger):
    """Fn.hstu_attention_fwd / _bwd on core_case's operands, element by element against the fp64 attention; ledger: the calling
    module's exact_check.Ledger"""
    import genrec_b200.functional as Fn
    from genrec_b200.hstu import _thresholds_on
    c = core_case(L, D, H, pos, time, seed)
    kind, npos, md = pos
    pb = pos_fixed(torch.arange(L), npos, md) if kind == "fix" else pos_fixed(-torch.arange(L), npos, md)
    uniform = bool((pb == pb[0]).all())
    ntime = time if isinstance(time, int) else 64
    meta = Fn.SeqMeta(c["pad"].to(torch.uint8).to(DEV), c["ts"].to(DEV) if c["ts"] is not None else None, pb.to(torch.uint8).to(DEV),
                      _thresholds_on(DEV), ntime, npos, (uniform, int(pb[0])))
    P, zp, dO = c["P"].to(DEV), c["zp"].to(DEV), c["dO"].to(DEV)
    wpos = c["wpos"].to(DEV)
    wtime = c["wtime"].to(DEV) if c["wtime"] is not None else None
    O = Fn.hstu_attention_fwd(P, meta, H, wpos, wtime, ntime)
    dzp, dpos, dtime = Fn.hstu_attention_bwd(P, zp, dO, meta, H, wpos, wtime, ntime)
    timed = wtime is not None and c["ts"] is not None
    w, masked, pbc, tbc = hr.cell_bias(meta.bias_index, wpos[int(pb[0]):int(pb[0]) + 1] if uniform else wpos, wtime if timed else None,
                                       1 if uniform else npos, H)
    valid = hr.causal_valid(c["pad"].to(DEV))
    assert torch.equal(masked, ~valid)
    at = hr.attention(P, w, valid, H, zp, dO)
    case = f"attn L{L}-D{D}-dh{D // H}-{kind}{npos}-t{time}"
    assert not bool(dzp[..., :D].any()), "the attention backward wrote the U columns"
    ledger.check(case, [("attn O", O, at["O"], at["a_O"]), ("attn dV", dzp[..., D:2 * D], at["dV"], at["a_dV"]),
                        ("attn dQ", dzp[..., 2 * D:3 * D], at["dQ"], at["a_dQ"]), ("attn dK", dzp[..., 3 * D:], at["dK"], at["a_dK"])])
    rows = torch.full_like(pbc, int(pb[0])) if uniform else pbc
    ref, mass, count = hr.table_sums(at["dS"], valid, rows[:, None], npos)
    assert table_excess(dpos, ref, mass.cpu(), count.cpu()) <= 1.0
    if timed:
        ref, mass, count = hr.table_sums(at["dS"], valid, tbc[:, None], wtime.shape[0])
        assert table_excess(dtime, ref, mass.cpu(), count.cpu()) <= 1.0


# ---------------------------------------------------------------------------------------------------- serving: cached extend, pool
SERVE_V, SERVE_NB = 500, 2


def _serve_model(D, H, use_time=True, seed=0, dropout=0.0):
    from genrec_b200.hstu import HSTU
    torch.manual_seed(seed)
    m = HSTU(SERVE_V, 64, D, H, SERVE_NB, dropout=dropout, use_temporal_bias=use_time)
    g = torch.Generator().manual_seed(seed + 100)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "attention_bias" in n:
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)
    return m.to("cuda").eval()


def _oracle_last(m, ids, ts):
    from oracle import hstu as oh
    sd = {k: v.detach().double().cpu() for k, v in m.state_dict().items()}
    logits, _ = oh.hstu_forward(ids.cpu(), ts.cpu() if ts is not None else None, None, sd, m.layers[0].num_heads, len(m.layers),
                                use_temporal_bias=m.use_temporal_bias)
    return logits[:, -1]


def _check_extend(ext, m, ids, ts, rows):
    """extend's logits of `rows` are as close to the fp64 oracle as last_logits on the same left-padded batch."""
    ref = _oracle_last(m, ids, ts)
    full = m.last_logits(ids, ts)
    e, b = relerr(ext[rows], ref[rows]), budget(full[rows], ref[rows])
    assert e <= b, (e, b)
    return full


def _sign_fixed(m):
    """Set the sign-fixed (non-uniform) position-bucket table through bucket_of_delta: bucket(i - j) instead of bucket(j - i)."""
    for layer in m.layers:
        rpb = layer.position_bias
        rpb._relative_position_bucket = (lambda f: (lambda rel: f(-rel)))(rpb._relative_position_bucket)
        rpb._table_cache.clear()
        rpb._uniform_cache.clear()


def _chunks(B, widths, seed, max_pad=3):
    """Per chunk of width w, user b's row holds min(b * max_pad, w - 1) left pads and then its next items."""
    g = torch.Generator().manual_seed(seed)
    chunks = []
    for w in widths:
        ids = torch.randint(1, SERVE_V + 1, (B, w), generator=g)
        ts = torch.randint(1, 3 * 86400, (B, w), generator=g)
        ts[:, ::3] = torch.randint(0, 30, (B, (w + 2) // 3), generator=g)
        for b in range(B):
            p = min(b * max_pad, w - 1)
            ids[b, :p] = 0
        chunks.append((ids, ts))
    return chunks


def _concat(chunks, upto):
    """left-padded [B, Lmax] batch of each user's items in the first `upto` chunks (timestamps made increasing per user)."""
    B = chunks[0][0].shape[0]
    rows_i, rows_t = [], []
    for b in range(B):
        items = torch.cat([c[0][b] for c in chunks[:upto]])
        gaps = torch.cat([c[1][b] for c in chunks[:upto]])
        keep = items != 0
        rows_i.append(items[keep])
        rows_t.append(gaps[keep])
    Lm = max(len(r) for r in rows_i)
    ids = torch.zeros(B, Lm, dtype=torch.int64)
    ts = torch.zeros(B, Lm, dtype=torch.int64)
    for b in range(B):
        n = len(rows_i[b])
        ids[b, Lm - n:] = rows_i[b]
        ts[b, Lm - n:] = rows_t[b]
    return ids, ts


def _absolute_ts(chunks):
    """turn the per-slot gaps into increasing timestamps per user, identically in chunk and concatenated form"""
    B = chunks[0][0].shape[0]
    last = torch.full((B,), 1_300_000_000, dtype=torch.int64)
    out = []
    for ids, gaps in chunks:
        ts = last[:, None] + torch.cumsum(gaps * (ids != 0), 1)
        ts[ids == 0] = 0
        last = torch.where((ids != 0).any(1), ts.max(1).values, last)
        out.append((ids, ts))
    return out


def _fill(m, pool, users, nfill, seed):
    """extend `users` by nfill items each (one call), to occupy pages"""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, SERVE_V + 1, (len(users), nfill), generator=g)
    ts = 1_200_000_000 + torch.cumsum(torch.randint(1, 86400, (len(users), nfill), generator=g), 1)
    m.extend_users(pool, torch.tensor(users), ids.cuda(), ts.cuda())


def _history_calls(nusers, ncalls, seed):
    """ncalls calls, each naming a different subset of users (B from 1 to nusers, random order) with a chunk of 1..9 slots per
    row, left-padded, some rows all padding.  Timestamps increase per user."""
    g = torch.Generator().manual_seed(seed)
    last = torch.full((nusers,), 1_300_000_000, dtype=torch.int64)
    calls = []
    for c in range(ncalls):
        B = 1 + c % nusers if c < nusers else int(torch.randint(1, nusers + 1, (1,), generator=g))
        users = torch.randperm(nusers, generator=g)[:B]
        w = int(torch.randint(1, 10, (1,), generator=g))
        ids = torch.randint(1, SERVE_V + 1, (B, w), generator=g)
        gaps = torch.randint(0, 2 * 86400, (B, w), generator=g)
        for r in range(B):
            pads = w if (c + r) % 5 == 3 else int(torch.randint(0, w, (1,), generator=g))
            ids[r, :pads] = 0
        ts = torch.zeros(B, w, dtype=torch.int64)
        for r in range(B):
            u = int(users[r])
            t = last[u] + torch.cumsum(gaps[r] * (ids[r] != 0), 0)
            ts[r] = torch.where(ids[r] != 0, t, torch.zeros_like(t))
            if (ids[r] != 0).any():
                last[u] = int(t[-1])
        calls.append((users, ids, ts))
    return calls


def _left_padded(hist, users):
    L = max(1, max(len(hist[int(u)][0]) for u in users))
    ids = torch.zeros(len(users), L, dtype=torch.int64)
    ts = torch.zeros(len(users), L, dtype=torch.int64)
    for r, u in enumerate(users.tolist()):
        n = len(hist[u][0])
        if n:
            ids[r, L - n:] = torch.tensor(hist[u][0])
            ts[r, L - n:] = torch.tensor(hist[u][1])
    return ids, ts


# ---------------------------------------------------------------------------------------------------- packed (jagged) batches
EDGE_LENGTHS = [0, 1, 63, 64, 65, 127, 128, 129, 200]


def _users(lengths, V, seed):
    """per-user histories (time order), timestamps and held-out targets -> the jagged device batch and hstu_collate_fn's input"""
    g = torch.Generator().manual_seed(seed)
    hist = [torch.randint(1, V + 1, (n,), generator=g) for n in lengths]
    stamps = [1_300_000_000 + torch.cumsum(torch.randint(1, 10 ** 6, (n,), generator=g), 0) for n in lengths]
    tgt = torch.randint(1, V + 1, (len(lengths),), generator=g)
    offsets = torch.zeros(len(lengths) + 1, dtype=torch.int64)
    offsets[1:] = torch.cumsum(torch.tensor(lengths, dtype=torch.int64), 0)
    items, ts = torch.cat(hist).long(), torch.cat(stamps).long()
    rows = [dict(history=h.tolist(), timestamps=s.tolist(), target=int(t)) for h, s, t in zip(hist, stamps, tgt)]
    return items.to(DEV), ts.to(DEV), offsets.to(DEV), tgt.to(DEV), rows


def run_block_jagged(lengths, D, H, pos, time, idle=5, seed=1, *, p=0.0, layer=0, seed_dev=None, max_len=None, offsets=None, lead=0, canary=0):
    """Forward and backward of one block through grb_hstu_layer_forward_jagged / _backward_jagged with a NaN-filled saved blob and
    workspace (its scratch for the ordered sums included).  pos: ("uni", bucket) or ("fix", npos, max_distance); time: buckets or "nots".  T = sum(lengths) + idle token rows;
    max_len defaults to the longest length.  lead: idle rows put in front of the batch (offsets[0] = lead, out of contract), the
    other rows' inputs unchanged.  offsets (a list of B + 1) replaces the device offsets (the kernels clamp it to [0, T)).  Rows
    outside [offsets[0], offsets[B]) are idle: pad, and dy = 0 there as the head gives it.  canary: rows of x, dy, y and dx past T
    in the same allocations, y / dx filled with 7.0.  -> the kernel's intermediates and gradients."""
    import genrec_b200.functional as Fn
    from genrec_b200 import _lib
    from genrec_b200._lib import HstuDims, HstuLayerGrads, HstuLayerParams, check, ptr, stream_ptr
    from genrec_b200.hstu import _thresholds_on
    lib = _lib.load()
    g = torch.Generator().manual_seed(seed)
    n_real = sum(lengths)
    Tm, B = n_real + idle, len(lengths)
    T = Tm + lead
    max_len = max_len or max(max(lengths), 1)
    off = torch.zeros(B + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(torch.tensor(lengths), 0)
    off += lead
    if offsets is not None:
        off = torch.tensor(offsets, dtype=torch.int64)
    lo, hi = min(max(int(off[0]), 0), T), min(max(int(off[-1]), 0), T)
    seq = torch.zeros(T, dtype=torch.bool)
    seq[lo:hi] = True
    ts = 1_300_000_000 + torch.cumsum(torch.randint(1, 3 * 86400, (Tm,), generator=g), 0)
    ts = torch.cat([torch.full((lead,), 1_300_000_000), ts])
    pad = (~seq).to(torch.uint8)
    uniform = pos[0] == "uni"
    npos = 8 if uniform else pos[1]
    pb = torch.full((max_len,), pos[1]) if uniform else pos_fixed(torch.arange(max_len), pos[1], pos[2])
    has_time = isinstance(time, int)
    ntime = time if has_time else 0
    offd = off.to(DEV)
    meta = Fn.SeqMeta(pad.to(DEV), ts.to(DEV) if has_time else None, pb.to(torch.uint8).to(DEV), _thresholds_on(DEV), ntime or 64, npos,
                      (uniform, int(pb[0])), offsets=offd, max_len=max_len)
    prm = _params(D, H, npos, ntime, seed + 7)
    xa = torch.randn(Tm + canary, D, generator=g)
    xa[:Tm:3] += 1000.0 * torch.where(torch.arange(0, Tm, 3) % 2 == 0, 1.0, -1.0)[:, None]   # LayerNorm's large-offset rows
    dya = torch.randint(-64, 65, (Tm + canary, D), generator=g).float() / 64
    xa = torch.cat([torch.randn(lead, D, generator=g), xa])
    dya = torch.cat([torch.zeros(lead, D), dya])
    dya[:T][~seq] = 0
    xa, dya = xa.to(DEV), dya.to(DEV)
    x, dy = xa[:T], dya[:T]
    sdev = None if seed_dev is None else torch.tensor([seed_dev], dtype=torch.int64, device=DEV)
    dseed = 0x1234_5678_9ABC_DEF0 + layer
    dims = HstuDims(B, max_len, D, H, npos, ntime, float(p), dseed, ptr(sdev), layer)
    names = ("proj_w", "proj_b", "pos_table", "time_table", "ln1_g", "ln1_b", "ffn1_w", "ffn1_b", "ffn2_w", "ffn2_b", "ln2_g", "ln2_b")
    pstruct = HstuLayerParams(*[ptr(prm[n]) if (n != "time_table" or has_time) else None for n in names])
    grads = {n: torch.zeros(prm[n].shape, dtype=torch.float32, device=DEV) for n in names}
    gstruct = HstuLayerGrads(*[ptr(grads[n]) for n in names])
    st_ = meta.struct()
    sl, wl = hr.saved_layout(T, D), hr.work_layout(T, D)
    nsaved, nwork = lib.grb_hstu_layer_saved_bytes_jagged(C.byref(dims), T), lib.grb_hstu_layer_workspace_bytes_jagged(C.byref(dims), T)
    assert nsaved == sl["bytes"] and wl["bytes"] <= nwork
    saved = torch.full((nsaved,), 0xFF, dtype=torch.uint8, device=DEV)        # NaN in bf16 and fp32
    ws = torch.full((nwork,), 0xFF, dtype=torch.uint8, device=DEV)   # the ordered sums' scratch too: a partial never stored shows
    ya, dxa = torch.full_like(xa, 7.0), torch.full_like(xa, 7.0)
    st = stream_ptr(DEV)
    check(lib.grb_hstu_layer_forward_jagged(C.byref(dims), C.byref(pstruct), C.byref(st_), ptr(offd), T, ptr(x), ptr(ya), ptr(saved), st))
    check(lib.grb_hstu_layer_backward_jagged(C.byref(dims), C.byref(pstruct), C.byref(st_), ptr(offd), T, ptr(dy), ptr(saved), ptr(dxa),
                                             C.byref(gstruct), ptr(ws), st))
    torch.cuda.synchronize()
    out = {n: hr.view(saved, sl, n) for n in sl if n != "bytes"}
    out.update({n: hr.view(ws, wl, n) for n in wl if n != "bytes"})
    out.update(grads=grads, prm=prm, meta=meta, off=[min(max(int(v), lo), hi) for v in off], D=D, H=H, n_real=n_real, T=T, x=x, dy=dy,
               y=ya[:T], dx=dxa[:T], y_canary=ya[T:], dx_canary=dxa[T:], seq=seq.to(DEV), uniform=uniform, npos=npos, pb0=int(pb[0]),
               has_time=has_time, ntime=ntime, p=p, layer=layer, seed=hr.effective_seed(dseed, p, seed_dev), max_len=max_len)
    return out


def attention_errors_jagged(r):
    """The attention of a packed block against hr.attention per sequence (the sequences of one length batched; on the GPU, in fp64),
    on the kernel's P, zp and dO.  Idle rows must hold O = 0 and dQ | dK | dV = 0.  -> ({O, dV, dQ, dK: worst error / allowance},
    {dpos, dtime: table_excess})"""
    D, H, prm, gr = r["D"], r["H"], r["prm"], r["grads"]
    for n in ("P", "O", "dO", "dzp", "y", "dx"):
        assert bool(torch.isfinite(r[n].float()).all()), f"{n} has an unwritten or non-finite element"
    seq = r["seq"]
    assert not bool(r["O"][~seq].any()) and not bool(r["dzp"][~seq][:, D:].any()), "idle rows of O / dQ dK dV are not zero"
    wpos = prm["pos_table"][r["pb0"]:r["pb0"] + 1] if r["uniform"] else prm["pos_table"]
    wtime = prm["time_table"][:r["ntime"]] if r["has_time"] else None
    nrows = 1 if r["uniform"] else r["npos"]
    acc = {"pos": None, "time": None}
    worst = {k: 0.0 for k in ("O", "dV", "dQ", "dK")}
    by_len = {}
    for b in range(len(r["off"]) - 1):
        lo, n = r["off"][b], min(r["off"][b + 1] - r["off"][b], r["max_len"])
        if n > 0:
            by_len.setdefault(n, []).append(lo)
    for n, starts in sorted(by_len.items()):
        step = max(1, (1 << 24) // (H * n * n))           # fp64 [seqs, H, n, n] tensors of at most 128 MB
        for c in range(0, len(starts), step):
            rows = (torch.tensor(starts[c:c + step])[:, None] + torch.arange(n)[None]).to(DEV)
            w, masked, pbc, tbc = hr.cell_bias(r["meta"].bias_index[rows], wpos, wtime, nrows, H)
            valid = hr.causal_valid(torch.zeros(rows.shape, dtype=torch.bool, device=DEV))
            assert torch.equal(masked, ~valid.expand_as(masked)), n
            at = hr.attention(r["P"][rows], w, valid, H, r["zp"][rows], r["dO"][rows])
            dzp = r["dzp"][rows]
            for name, got, ref, allow in [("O", r["O"][rows], at["O"], at["a_O"]), ("dV", dzp[..., D:2 * D], at["dV"], at["a_dV"]),
                                          ("dQ", dzp[..., 2 * D:3 * D], at["dQ"], at["a_dQ"]), ("dK", dzp[..., 3 * D:], at["dK"], at["a_dK"])]:
                worst[name] = max(worst[name], dr.worst(got, ref, allow))
            bucket = torch.full_like(pbc, r["pb0"]) if r["uniform"] else pbc
            parts = {"pos": hr.table_sums(at["dS"], valid, bucket[:, None], r["npos"])}
            if r["has_time"]:
                parts["time"] = hr.table_sums(at["dS"], valid, tbc[:, None], r["ntime"])
            for k, v in parts.items():
                acc[k] = v if acc[k] is None else tuple(a + e for a, e in zip(acc[k], v))
            del at, w, masked, valid
    excess = {}
    for k, name, table in (("pos", "dpos", "pos_table"), ("time", "dtime", "time_table")):
        if acc[k] is not None:
            ref, mass, count = acc[k]
            excess[name] = table_excess(gr[table], ref, mass.cpu(), count.cpu())
        else:                                             # no time term, or no sequence at all
            assert not bool(gr[table].any()), f"{table} gradient without a live cell"
    return worst, excess


def _jagged_model(V, blocks=2, D=64, H=2, seed=0, fixed=False):
    from genrec_b200.hstu import HSTU
    torch.manual_seed(seed)
    m = HSTU(V, 200, D, H, blocks, dropout=0.0).to(DEV).train()
    if fixed:
        sign_fix(m)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if "attention_bias" in n:
                p.normal_(0, 0.3)
    return m


# ---------------------------------------------------------------------------------------------------- the headline (cfg2) model
# BASELINE.json configs[1]: HSTU 4 blocks, d=128, h=4, seq_len=200, V=12,101
CFG2_V, CFG2_L, CFG2_D, CFG2_H, CFG2_NB = 12101, 200, 128, 4, 4


def _cfg2_model(seed=0, dropout=0.0):
    from genrec_b200.hstu import HSTU
    torch.manual_seed(seed)
    m = HSTU(CFG2_V, CFG2_L, CFG2_D, CFG2_H, CFG2_NB, dropout=dropout)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():                      # leave the reference init but make every term matter
        for n, p in m.named_parameters():
            if "attention_bias" in n:
                p.copy_(0.3 * torch.randn(p.shape, generator=g))
            elif n.endswith("bias") and p.dim() == 1:
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
            elif "norm" in n and n.endswith("weight"):
                p.add_(0.1 * torch.randn(p.shape, generator=g))
            elif "item_embedding" in n:
                p.mul_(10.0)
                p[0].zero_()
            elif p.dim() == 2:
                p.mul_(3.0)
    return m


def _oracle_run(ids, ts, tg, sd, autocast):
    """Oracle forward + backward on the host cores; returns loss, parameter grads and the gradient entering the last block."""
    from oracle import hstu as oh
    p = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    grabbed = {}
    orig = oh.hstu_layer_forward

    def spy(x, *a, **kw):
        if a[3] == f"layers.{CFG2_NB - 1}.":
            x.retain_grad(); grabbed["x_last"] = x
        return orig(x, *a, **kw)

    oh.hstu_layer_forward = spy
    try:
        if autocast:
            with torch.autocast("cpu", dtype=torch.bfloat16):
                _, lo = oh.hstu_forward(ids, ts, tg, p, CFG2_H, CFG2_NB)
            lo.float().backward()
        else:
            _, lo = oh.hstu_forward(ids, ts, tg, p, CFG2_H, CFG2_NB)
            lo.backward()
    finally:
        oh.hstu_layer_forward = orig
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    return float(lo), grads, grabbed["x_last"].grad.float()


# ---------------------------------------------------------------------------------------------------- Recall@10 users
def markov_users(num_users, V, L, seed, clusters=10):
    """First-order Markov chain over item clusters: the next item is (mostly) drawn from the successor cluster, so the task is
    learnable and Recall@10 is far above chance."""
    g = torch.Generator().manual_seed(seed)
    per = V // clusters
    seqs, stamps = [], []
    for _ in range(num_users):
        c = int(torch.randint(0, clusters, (1,), generator=g))
        items, ts, t = [], [], 1_300_000_000
        for _ in range(L + 1):
            if float(torch.rand(1, generator=g)) < 0.9:
                c = (c + 1) % clusters
            else:
                c = int(torch.randint(0, clusters, (1,), generator=g))
            items.append(1 + c * per + int(torch.randint(0, per, (1,), generator=g)))
            t += int(torch.randint(60, 86400, (1,), generator=g))
            ts.append(t)
        seqs.append(items); stamps.append(ts)
    return torch.tensor(seqs), torch.tensor(stamps)
