"""HSTU attention across its bias-table configurations, against fp64 restatements and the fp64 oracle.

Position tables: the reference's (bucket(j - i) clamped at 0: every causal cell in bucket 0, one uniform row), a uniform row other
than 0, and the sign-fixed T5 table bucket(i - j) with 8, 16, 32 or 64 buckets and a max_position_distance below L, so that the
clamped top bucket is hit.  Time tables: 1, 20, 63 or 64 buckets, no table, or no timestamps.  Every batch holds a mid-sequence pad,
a left-padded row, a fully padded row and a row whose timestamps span 9.15e18 (time bucket 63, the top of an int64 difference).

The cases, restatements and tolerances live in hstu_cases.py, shared with test_hstu_bias_configs_cpu.py, which checks that each
tolerance fails a model restated with wrong bucket logic.
"""
import pytest
import torch

from tests.hstu_cases import (CORE_CASES, F32_LAYER_CASES, F32_TOL, LAYER_CASES, SERVE_V, _absolute_ts, _chunks, _concat, _history_calls,
                              _left_padded, batch, cell_buckets, core_case, core_excess, core_id, core_reference, layer_case, layer_excess,
                              oracle_layer, patch_oracle, pos_fixed, randomise, sign_fix)
from tests.util import relerr

pytestmark = pytest.mark.gpu

# HSTU (bf16 path) against the fp64 oracle: the tolerances of test_hstu_gpu.py::test_layer_vs_oracle_shapes
MODEL_LOSS_TOL = 1e-2          # |loss - loss_ref| / |loss_ref|
MODEL_GRAD_TOL = 5e-2
LAST_LOGITS_TOL = 2e-2         # last_logits / extend / extend_users against the fp64 oracle


# ---------------------------------------------------------------------------------------------------- attention core


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
    c = model_case(64, 64, 2, 2, 16, 40, 20, seed=13, num_items=SERVE_V)
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
