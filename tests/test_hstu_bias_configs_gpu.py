"""HSTU attention across its bias-table configurations, against fp64 restatements and the fp64 oracle.

Position tables: the reference's (bucket(j - i) clamped at 0: every causal cell in bucket 0, one uniform row), a uniform row other
than 0, and the sign-fixed T5 table bucket(i - j) with 8, 16, 32 or 64 buckets and a max_position_distance below L, so that the
clamped top bucket is hit.  Time tables: 1, 20, 63 or 64 buckets, no table, or no timestamps.  Every batch holds a mid-sequence pad,
a left-padded row, a fully padded row and a row whose timestamps span 9.15e18 (time bucket 63, the top of an int64 difference).

The helpers and tolerances here are shared with test_hstu_bias_configs_cpu.py, which checks that each tolerance fails a model
restated with wrong bucket logic.
"""
import pytest
import torch
import torch.nn.functional as F

from tests.util import relerr

pytestmark = pytest.mark.gpu

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
# HSTULayer / HSTU (bf16 path) against the fp64 oracle: the tolerances of test_hstu_gpu.py::test_layer_vs_oracle_shapes
LAYER_Y_TOL = 2.5e-2
LAYER_DX_TOL = 2.5e-2
LAYER_GRAD_TOL = 4e-2
MODEL_LOSS_TOL = 1e-2          # |loss - loss_ref| / |loss_ref|
MODEL_GRAD_TOL = 5e-2
LAST_LOGITS_TOL = 2e-2         # last_logits / extend / extend_users against the fp64 oracle
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


def _meta(c, pos_bucket, dev):
    import genrec_b200.functional as Fn
    from genrec_b200.hstu import _thresholds_on
    npos = c["pos"][1]
    ntime = c["time"] if isinstance(c["time"], int) else 64
    pb = pos_bucket.to(torch.uint8)
    return Fn.SeqMeta(c["pad"].to(torch.uint8).to(dev), c["ts"].to(dev) if c["ts"] is not None else None, pb.to(dev),
                      _thresholds_on(dev), ntime, npos, (bool((pb == pb[0]).all()), int(pb[0])))


def run_core(c, pos_bucket=None):
    """the kernels on case c: O, dzp, dpos, dtime (CPU).  pos_bucket: the [L] table of delta = i - j (default: c's rule)."""
    import genrec_b200.functional as Fn
    dev = torch.device("cuda:0")
    if pos_bucket is None:
        pos_bucket = cell_buckets(c)[0][:, 0]           # column j = 0: delta = i
    meta = _meta(c, pos_bucket, dev)
    ntime = c["time"] if isinstance(c["time"], int) else 64
    P, zp, dO = c["P"].to(dev), c["zp"].to(dev), c["dO"].to(dev)
    wpos = c["wpos"].to(dev)
    wtime = c["wtime"].to(dev) if c["wtime"] is not None else None
    O = Fn.hstu_attention_fwd(P, meta, c["H"], wpos, wtime, ntime)
    dzp, dpos, dtime = Fn.hstu_attention_bwd(P, zp, dO, meta, c["H"], wpos, wtime, ntime)
    torch.cuda.synchronize()
    return dict(O=O.float().cpu(), dzp=dzp.float().cpu(), dpos=dpos.cpu(), dtime=dtime.cpu() if dtime is not None else None)


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


# ---------------------------------------------------------------------------------------------------- (a) bias index
@pytest.mark.parametrize("L", [7, 200])
@pytest.mark.parametrize("npos,md", [(8, 12), (32, 100), (64, 80)])
def test_bias_index_bit_exact_non_uniform(L, npos, md):
    """hstu_bias_index_kernel: pb(i - j) * 64 + tb on valid cells, npos * 64 on masked ones, for every time-bucket count."""
    dev = torch.device("cuda:0")
    for time in (1, 20, 63, 64, "nots"):
        c = core_case(L, 64, 2, ("fix", npos, md), time, seed=L + npos)
        pb, tb = cell_buckets(c)
        assert not bool((pb[:, 0] == pb[0, 0]).all())            # really the per-bucket layout
        m = _meta(c, pb[:, 0], dev)
        got = m.bias_index.cpu().to(torch.int32) & 0xFFFF
        want = pb[None] * 64 + (tb if tb is not None else 0)
        ii = torch.arange(L)
        valid = (ii[None, :] <= ii[:, None])[None] & ~c["pad"][:, None, :]
        want = torch.where(valid, want, torch.full_like(want, npos * 64)).to(torch.int32)
        assert torch.equal(got[:, :, :L], want), (time, (got[:, :, :L] != want).nonzero()[:5])


# ---------------------------------------------------------------------------------------------------- (b) attention core
@pytest.mark.parametrize("case", CORE_CASES, ids=core_id)
def test_attention_core_vs_fp64(case):
    L, D, H, pos, time = case
    c = core_case(L, D, H, pos, time, seed=L * 7 + D + H)
    pb, tb = cell_buckets(c)
    got = run_core(c)
    ref = core_reference(c, pb, tb)
    assert torch.isfinite(got["O"]).all() and torch.isfinite(got["dzp"]).all()
    assert got["O"][2].abs().max() == 0                                  # fully padded sequence: exact zeros
    assert got["dzp"][..., :D].abs().max() == 0                          # the U columns belong to the gate's backward
    assert (got["dtime"] is None) == (ref["dtime"] is None)
    ex = core_excess(got, ref, pb, tb, D)
    assert max(ex.values()) <= 1.0, ex


# ---------------------------------------------------------------------------------------------------- (c) uniform bucket 7
@pytest.mark.parametrize("time", [20, "nots"])
def test_uniform_position_bucket_other_than_zero(time):
    """A constant table of bucket 7: the forward reads row 7 and only row 7 receives gradient."""
    L, D, H = 130, 128, 4
    c = core_case(L, D, H, ("fix", 32, 100), time, seed=71)
    pb = torch.full((L, L), 7, dtype=torch.long)
    tb = cell_buckets(c)[1]
    got = run_core(c, pos_bucket=torch.full((L,), 7))
    ref = core_reference(c, pb, tb)
    ex = core_excess(got, ref, pb, tb, D)
    assert max(ex.values()) <= 1.0, ex
    assert got["dpos"][7].abs().min() > 0
    assert got["dpos"][:7].abs().max() == 0 and got["dpos"][8:].abs().max() == 0
    # the forward reads row 7: moving row 0 changes nothing, moving row 7 changes O
    c0 = dict(c, wpos=c["wpos"].clone())
    c0["wpos"][0] += 1.0
    assert torch.equal(run_core(c0, pos_bucket=torch.full((L,), 7))["O"], got["O"])
    c7 = dict(c, wpos=c["wpos"].clone())
    c7["wpos"][7] += 1.0
    assert not torch.equal(run_core(c7, pos_bucket=torch.full((L,), 7))["O"], got["O"])


# ---------------------------------------------------------------------------------------------------- (d) HSTULayer
# (B = 4, L, D, H, npos, md, ntime): sign-fixed buckets
LAYER_CASES = [(200, 128, 4, 16, 40, 20), (65, 128, 2, 64, 80, 63), (257, 128, 4, 64, 80, 20), (130, 128, 2, 16, 40, 63)]


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


@pytest.mark.parametrize("case", LAYER_CASES, ids=lambda c: "L{}-dh{}-npos{}-t{}".format(c[0], c[1] // c[2], c[3], c[5]))
def test_layer_vs_oracle_sign_fixed(case, monkeypatch):
    patch_oracle(monkeypatch, pos_fixed)
    c = layer_case(*case, seed=case[0] + case[3])
    ref = oracle_layer(c)
    dev = torch.device("cuda:0")
    layer = c["layer"].to(dev).train()
    sign_fix(layer)
    assert not layer.position_bias.uniform_of(case[0], dev)[0]
    x = c["x"].to(dev).requires_grad_(True)
    y = layer(x, None, c["pad"].to(dev), c["ts"].to(dev))
    y.backward(c["dy"].to(dev))
    ex = layer_excess(y, x.grad, {n: p.grad for n, p in layer.named_parameters()}, ref)
    assert max(ex.values()) <= 1.0, ex


# ---------------------------------------------------------------------------------------------------- (e) HSTU training step
def model_case(L, D, H, NB, npos, md, ntime, seed, num_items=300):
    from genrec_b200.hstu import HSTU
    torch.manual_seed(seed)
    m = HSTU(num_items, L, D, H, NB, dropout=0.0, num_position_buckets=npos, num_time_buckets=ntime, max_position_distance=md)
    randomise(m, seed)
    ids, ts, pad = batch(L, seed, num_items)
    g = torch.Generator().manual_seed(seed + 2)
    tg = torch.randint(1, num_items + 1, (4, L), generator=g)
    tg[pad] = 0
    return dict(model=m, sd={k: v.detach().clone() for k, v in m.state_dict().items()}, ids=ids, ts=ts, tg=tg, H=H, NB=NB, npos=npos,
                md=md)


def oracle_model(c, targets=True):
    from oracle import hstu as oh
    sd = {k: v.double().requires_grad_(targets) for k, v in c["sd"].items()}
    logits, loss = oh.hstu_forward(c["ids"], c["ts"], c["tg"] if targets else None, sd, c["H"], c["NB"], True, c["npos"], c["md"])
    if not targets:
        return logits.detach(), None, None
    loss.backward()
    return logits.detach(), loss.detach(), {k: v.grad for k, v in sd.items()}


def test_model_training_step_vs_oracle(monkeypatch):
    patch_oracle(monkeypatch, pos_fixed)
    c = model_case(130, 64, 2, 2, 16, 40, 20, seed=5)
    _, loss_ref, grads_ref = oracle_model(c)
    dev = torch.device("cuda:0")
    m = c["model"].to(dev).train()
    sign_fix(m)
    _, loss = m(c["ids"].to(dev), c["ts"].to(dev), c["tg"].to(dev))
    loss.backward()
    assert abs(loss.item() - loss_ref.item()) <= MODEL_LOSS_TOL * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    for n, p in m.named_parameters():
        ref = grads_ref[n]
        got = p.grad if p.grad is not None else torch.zeros_like(p)
        assert relerr(got, ref) <= MODEL_GRAD_TOL, (n, relerr(got, ref))


def test_custom_op_block_equals_module_block_20_time_buckets():
    """torch.ops.genrec_b200.hstu_layer == HSTULayer with num_time_buckets = 20 (the custom op takes uniform position buckets)."""
    import genrec_b200.ops  # noqa: F401
    from genrec_b200.hstu import _thresholds_on
    dev = torch.device("cuda:0")
    c = layer_case(70, 128, 4, 32, 128, 20, seed=9)
    layer = c["layer"].to(dev).train()
    pad, ts = c["pad"].to(dev), c["ts"].to(dev)
    x, dy = c["x"].to(dev), c["dy"].to(dev)
    xi = x.clone().requires_grad_(True)
    y = layer(xi, None, pad, ts)
    y.backward(dy)
    ref = (y.detach().clone(), xi.grad.clone(), [p.grad.clone() for p in layer._params()])
    layer.zero_grad(set_to_none=True)
    pad8 = pad.to(torch.uint8)
    xj = x.clone().requires_grad_(True)
    y2, _saved = torch.ops.genrec_b200.hstu_layer(xj, pad8, ts, _thresholds_on(dev), *layer._params(), c["H"], 20, 0, 0.0, 0, None, 0)
    y2.backward(dy)
    torch.testing.assert_close(y2, ref[0], rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(xj.grad, ref[1], rtol=1e-4, atol=1e-5)
    for p, g in zip(layer._params(), ref[2]):
        torch.testing.assert_close(p.grad, g, rtol=2e-3, atol=1e-4 * max(1.0, g.abs().max().item()))


# ---------------------------------------------------------------------------------------------------- (f) fp32-exact forward
F32_LAYER_CASES = [(130, 128, 4, 16, 40, 20), (200, 128, 2, 64, 80, 64), (65, 64, 2, 32, 100, 20)]


@pytest.mark.parametrize("case", F32_LAYER_CASES, ids=lambda c: "L{}-dh{}-npos{}-t{}".format(c[0], c[1] // c[2], c[3], c[5]))
def test_layer_fp32_vs_oracle_sign_fixed(case, monkeypatch):
    patch_oracle(monkeypatch, pos_fixed)
    c = layer_case(*case, seed=case[0] + 3)
    yo, _, _ = oracle_layer(c, with_grad=False)
    dev = torch.device("cuda:0")
    layer = c["layer"].to(dev).eval()
    sign_fix(layer)
    layer.precision = "fp32"
    with torch.no_grad():
        y = layer(c["x"].to(dev), None, c["pad"].to(dev), c["ts"].to(dev))
    assert relerr(y, yo) < F32_TOL, relerr(y, yo)


@pytest.mark.parametrize("ntime", [20, 64])
def test_model_fp32_vs_oracle_sign_fixed(ntime, monkeypatch):
    patch_oracle(monkeypatch, pos_fixed)
    c = model_case(100, 64, 2, 2, 16, 40, ntime, seed=ntime)
    logits_ref, _, _ = oracle_model(c, targets=False)
    dev = torch.device("cuda:0")
    m = c["model"].to(dev).eval().set_precision("fp32")
    sign_fix(m)
    with torch.no_grad():
        logits, _ = m(c["ids"].to(dev), c["ts"].to(dev))
        last = m.last_logits(c["ids"].to(dev), c["ts"].to(dev))
    assert relerr(logits, logits_ref) < F32_TOL, relerr(logits, logits_ref)
    assert relerr(last, logits_ref[:, -1]) < F32_TOL, relerr(last, logits_ref[:, -1])


# ---------------------------------------------------------------------------------------------------- (g) last_logits, extend
def _serving_model():
    """2 blocks, D = 64, H = 2, 16 sign-fixed position buckets (max distance 40), 20 time buckets, 500 items."""
    from tests.test_hstu_extend_gpu import V
    c = model_case(64, 64, 2, 2, 16, 40, 20, seed=13, num_items=V)
    m = c["model"].to("cuda").eval()
    sign_fix(m)
    return m, c


def _oracle_last(m, c, ids, ts):
    return oracle_model(dict(c, sd={k: v.detach().cpu() for k, v in m.state_dict().items()}, ids=ids.cpu(), ts=ts.cpu()),
                        targets=False)[0][:, -1]


@pytest.mark.parametrize("L", [1, 65, 200])
def test_last_logits_vs_oracle(L, monkeypatch):
    patch_oracle(monkeypatch, pos_fixed)
    m, c = _serving_model()
    ids, ts, _ = batch(L, seed=L)
    got = m.last_logits(ids.cuda(), ts.cuda())
    ref = _oracle_last(m, c, ids, ts)
    rows = [0, 1, 3] if L > 1 else [0, 3]          # row 2 is all padding; at L = 1 so is row 0
    assert relerr(got[rows], ref[rows]) <= LAST_LOGITS_TOL, relerr(got[rows], ref[rows])


def test_extend_vs_oracle(monkeypatch):
    from tests.test_hstu_extend_gpu import _absolute_ts, _chunks, _concat
    patch_oracle(monkeypatch, pos_fixed)
    m, c = _serving_model()
    B, widths = 3, [1, 7, 64, 65, 63]
    chunks = _absolute_ts(_chunks(B, widths, seed=23))
    st = m.new_state(B, sum(widths))
    for k, (ids, ts) in enumerate(chunks):
        ext = m.extend(st, ids.cuda(), ts.cuda())
        cids, cts = _concat(chunks, k + 1)
        ref = _oracle_last(m, c, cids, cts)
        assert relerr(ext, ref) <= LAST_LOGITS_TOL, (k, relerr(ext, ref))


def test_extend_users_vs_oracle(monkeypatch):
    from tests.test_hstu_pool_gpu import _history_calls, _left_padded
    patch_oracle(monkeypatch, pos_fixed)
    m, c = _serving_model()
    nusers = 6
    pool = m.new_pool(max_users=nusers, num_pages=3 * nusers, page_size=64, max_items=192)
    hist = {u: ([], []) for u in range(nusers)}
    for users, ids, ts in _history_calls(nusers, 12, seed=29):
        out = m.extend_users(pool, users, ids.cuda(), ts.cuda())
        for r, u in enumerate(users.tolist()):
            keep = ids[r] != 0
            hist[u][0].extend(ids[r][keep].tolist())
            hist[u][1].extend(ts[r][keep].tolist())
        rows = [r for r, u in enumerate(users.tolist()) if hist[u][0]]
        if rows:
            cids, cts = _left_padded(hist, users)
            ref = _oracle_last(m, c, cids, cts)
            assert relerr(out[rows], ref[rows]) <= LAST_LOGITS_TOL, relerr(out[rows], ref[rows])


# ---------------------------------------------------------------------------------------------------- (h) determinism
@pytest.mark.parametrize("ntime", [20, 64])
@pytest.mark.parametrize("pos", [("ref", 32, 128), ("fix", 64, 80)])
def test_backward_is_bit_identical_across_runs(ntime, pos):
    """dzp and both table gradients are bit-identical run to run (lost or racing histogram updates would break this)."""
    c = core_case(257, 128, 4, pos, ntime, seed=ntime + pos[1])
    a, b = run_core(c), run_core(c)
    for k in ("dzp", "dpos", "dtime"):
        assert torch.equal(a[k], b[k]), k
