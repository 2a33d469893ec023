"""The tied-embedding cross-entropy head on the H100 against the fp64 reference of tests/head_reference.py, which rounds where the
kernels round: every dispatch path (the fused wgmma kernels at D = 64 / 128, the stored-logits vector kernel at D = 256 with
C <= 16384 and the scalar kernel above), token and class counts on both sides of the 64- and 128-wide tiles, the benchmark
shapes and the two logit-range cases.  Then the contracts of the C ABI (gradients accumulate into dtable / dln_g / dln_b, dx is
overwritten, the workspace may hold garbage, a loss-only call, repeat calls, the grad-sink paths, unaligned targets, an all-ignored
batch), grb_head_logits and grb_eval_rank_metrics.  `pytest -s` prints the measured errors of every case as one table."""
import math

import pytest
import torch

from tests.head_cases import EPS, _call, _dev, _reference, _to_dev
from tests.head_reference import LOSS_FLOOR, TOL, format_table, head_errors, make_case, violations

pytestmark = pytest.mark.gpu

TOKENS = (1, 63, 64, 65, 127, 128, 129, 385)
# logits of grb_head_logits: |error| <= TOL_LOGITS * (|xf| |E|^T), fp32 accumulation of exact bf16 products.  Measured 1.9e-7 on an
# H100 80GB HBM3 (700 W power limit).
TOL_LOGITS = 6e-7
_ROWS = []
_LOGITS = []


@pytest.fixture(scope="module", autouse=True)
def _error_table():
    yield
    if _ROWS:
        head = format_table("", {k: 0.0 for k in list(TOL) + ["ignored dx"]})[0]
        print("\n" + head + "\n|" + "---|" * (len(TOL) + 2))
        print("\n".join(line for _, line in _ROWS))
        worst = {k: max(e[k] for e, _ in _ROWS) for k in list(TOL) + ["ignored dx"]}
        print(format_table("max over all cases", worst)[1])
    if _LOGITS:
        print(f"grb_head_logits, {len(_LOGITS)} cases: max |error| / (|xf| |E|^T) = {max(e for e, _ in _LOGITS):.2e}, "
              f"loss of these logits vs the fused loss = {max(e for _, e in _LOGITS):.2e}")


def _check(name, T, D, C, kind="plain", seed=None):
    c = _to_dev(make_case(T, D, C, seed=T * 1009 + C * 7 + D if seed is None else seed, kind=kind))
    got = _call(c)
    err = head_errors(got, _reference(c), c["tg"])
    _ROWS.append((err, format_table(name, err)[1]))
    assert not violations(err), (name, violations(err), err)


# ------------------------------------------------------------------------------------------------ every dispatch path
@pytest.mark.parametrize("T", TOKENS)
@pytest.mark.parametrize("C", (2, 63, 64, 65, 129, 1203, 12102))
@pytest.mark.parametrize("D", (64, 128))
def test_fused_head_vs_fp64(D, C, T):
    _check(f"fused D={D} C={C} T={T}", T, D, C)


@pytest.mark.parametrize("T", TOKENS)
@pytest.mark.parametrize("C", (65, 12102, 16384, 16385, 40001))
def test_stored_logits_head_vs_fp64(C, T):
    """D = 256: GEMM + ce_fwd_bwd_vec_kernel<8> up to C = 16384, GEMM + the scalar ce_fwd_bwd_kernel above."""
    _check(f"stored D=256 C={C} T={T}", T, 256, C)


@pytest.mark.parametrize("cfg,T,D", [("cfg2", 25600, 128), ("cfg3", 65536, 256)])
def test_benchmark_shapes_vs_fp64(cfg, T, D):
    _check(f"{cfg} T={T} D={D} C=12102", T, D, 12102)


@pytest.mark.parametrize("D", (64, 128, 256))
@pytest.mark.parametrize("kind,C", [("wide", 3000), ("overflow", 3000), ("small", 65)])
def test_logit_range_vs_fp64(kind, C, D):
    """wide: logits over +-60 nats; overflow: one class ~1.5 D nats above every other logit; small: logits within a few nats, where
    a padding column entering the softmax would carry real mass."""
    _check(f"{kind} D={D} C={C} T=385", 385, D, C, kind=kind)


# ------------------------------------------------------------------------------------------------ contracts of the C ABI
CONTRACT_SHAPES = [(385, 64, 129), (385, 128, 1203), (385, 256, 1203), (385, 256, 16385)]


def _ulp_close(a, b, scale):
    """|a - b| <= 4 fp32 ulps of `scale` (elementwise)"""
    return bool(((a - b).abs() <= 4 * 2.0 ** -23 * scale.abs() + 1e-30).all())


@pytest.mark.parametrize("T,D,C", CONTRACT_SHAPES)
def test_gradients_accumulate_and_dx_is_overwritten(T, D, C):
    c = _to_dev(make_case(T, D, C, seed=11))
    fresh = _call(c)
    g = torch.Generator(device=_dev()).manual_seed(3)
    A = {k: torch.randn(v.shape, device=_dev(), generator=g) * v.abs().max() for k, v in fresh.items() if k in ("dE", "dg", "db")}
    got = _call(c, dx=torch.full_like(c["x"], float("nan")), dtable=A["dE"].clone(), dg=A["dg"].clone(), db=A["db"].clone())
    assert torch.equal(got["dx"], fresh["dx"])
    assert got["loss"] == fresh["loss"]
    for k in ("dE", "dg", "db"):
        assert _ulp_close(got[k], A[k] + fresh[k], A[k].abs() + fresh[k].abs()), k


@pytest.mark.parametrize("T,D,C", CONTRACT_SHAPES)
def test_workspace_garbage_gives_the_same_bits(T, D, C):
    from genrec_b200 import _lib
    c = _to_dev(make_case(T, D, C, seed=12))
    clean = _call(c)
    ws = torch.full((_lib.load().grb_head_workspace_bytes(T, D, C),), 0xFF, dtype=torch.uint8, device=_dev())
    dirty = _call(c, ws=ws)
    assert dirty["loss"] == clean["loss"]
    for k in ("dx", "dg", "db", "dE"):
        assert torch.equal(dirty[k], clean[k]), k


@pytest.mark.parametrize("T,D,C", CONTRACT_SHAPES)
def test_loss_only_call_gives_the_same_loss(T, D, C):
    c = _to_dev(make_case(T, D, C, seed=13))
    assert _call(c, loss_only=True)["loss"] == _call(c)["loss"]


@pytest.mark.parametrize("T,D,C", CONTRACT_SHAPES)
def test_unaligned_targets_give_the_same_results(T, D, C):
    """targets at an 8-byte offset: ce_count_kernel counts them without its 16-byte loads"""
    c = _to_dev(make_case(T, D, C, seed=14))
    store = torch.empty(T + 1, dtype=torch.int64, device=_dev())
    tg = store[1:]
    tg.copy_(c["tg"])
    assert tg.data_ptr() % 16 == 8
    a, b = _call(c), _call(c, tg=tg)
    assert a["loss"] == b["loss"]
    for k in ("dx", "dg", "db", "dE"):
        assert torch.equal(a[k], b[k]), k


def test_repeat_calls_are_bit_identical_at_cfg2_with_and_without_deferred_weight_gradients():
    from genrec_b200 import _lib
    from genrec_b200._lib import check, stream_ptr
    lib = _lib.load()
    c = _to_dev(make_case(25600, 128, 12102, seed=15))
    runs = [_call(c), _call(c)]
    try:
        check(lib.grb_set_defer_weight_grads(1))
        for _ in range(2):
            r = _call(c)
            check(lib.grb_join_deferred(stream_ptr(_dev())))
            torch.cuda.synchronize()
            runs.append(r)
    finally:
        check(lib.grb_set_defer_weight_grads(0))
        check(lib.grb_join_deferred(stream_ptr(_dev())))
    for r in runs[1:]:
        assert r["loss"] == runs[0]["loss"]
        for k in ("dx", "dg", "db", "dE"):
            assert torch.equal(r[k], runs[0][k]), k


@pytest.mark.parametrize("D", (64, 128, 256))
def test_head_loss_fn_scales_by_dloss_and_the_direct_sink_gives_the_same_bits(D):
    from genrec_b200 import functional as Fn
    c = _to_dev(make_case(2 * 97, D, 1203, seed=16))
    x3, tg2 = c["x"].view(2, 97, D), c["tg"].view(2, 97)

    def leaves():
        return [t.clone().requires_grad_(True) for t in (x3, c["ln_g"], c["ln_b"], c["table"])]

    def grads(ts):
        return [t.grad for t in ts]

    unit = leaves()
    Fn.HeadLossFn.apply(*unit, c["tb"], tg2, EPS).backward()
    scaled = leaves()
    dloss = torch.tensor(0.37, device=_dev())
    Fn.HeadLossFn.apply(*scaled, c["tb"], tg2, EPS).backward(dloss)
    for a, b in zip(grads(scaled), grads(unit)):
        assert torch.equal(a, b * dloss)
    direct = leaves()
    sink = (torch.zeros(D, device=_dev()), torch.zeros(D, device=_dev()), torch.zeros(1203, D, device=_dev()))
    Fn.HeadLossFn.apply(*direct, c["tb"], tg2, EPS, sink, True).backward()
    torch.cuda.synchronize()
    assert torch.equal(direct[0].grad, unit[0].grad)
    for s, u in zip(sink, grads(unit)[1:]):
        assert torch.equal(s, u)


@pytest.mark.parametrize("D,C", [(64, 129), (128, 1203), (256, 1203), (256, 16385)])
def test_all_rows_ignored_gives_nan_loss_and_zero_gradients(D, C):
    c = _to_dev(make_case(130, D, C, seed=17))
    c["tg"].zero_()
    got = _call(c)
    assert math.isnan(got["loss"])
    for k in ("dx", "dg", "db", "dE"):
        assert got[k].abs().max().item() == 0, k


# ------------------------------------------------------------------------------------------------ grb_head_logits
@pytest.mark.parametrize("T", (1, 129))
@pytest.mark.parametrize("C", (2, 65, 12102))
@pytest.mark.parametrize("D", (64, 128, 256))
def test_head_logits_vs_fp64(D, C, T):
    from genrec_b200 import functional as Fn
    c = _to_dev(make_case(T, D, C, seed=18 + C + T))
    logits = Fn.head_logits(c["x"][None], c["ln_g"], c["ln_b"], c["table"], c["tb"], EPS)[0]
    xf, _, _ = Fn.layernorm_fwd(c["x"], c["ln_g"], c["ln_b"], EPS)
    X, E = xf.double(), c["tb"].double()
    ref = X @ E.t()
    bound = X.abs() @ E.abs().t()
    assert logits.shape == (T, C)
    err = ((logits.double() - ref).abs() / bound.clamp_min(1e-30)).max().item()
    # the fp64 loss of these logits is the loss of the fused head
    tg = c["tg"]
    lse = torch.logsumexp(logits.double(), 1)
    loss = ((lse - logits.double().gather(1, tg[:, None])[:, 0])[tg != 0]).mean().item()
    fused = _call(c, loss_only=True)["loss"]
    lerr = abs(fused - loss) / max(abs(loss), LOSS_FLOOR)
    _LOGITS.append((err, lerr))
    assert err <= TOL_LOGITS, err
    assert lerr <= TOL["loss"], (fused, loss)


# ------------------------------------------------------------------------------------------------ grb_eval_rank_metrics
def test_eval_rank_metrics_exact_ranks_with_ties_and_skipped_targets():
    from genrec_b200 import functional as Fn
    B, C = 4096, 12102
    g = torch.Generator().manual_seed(19)
    lg = torch.randn(B, C, generator=g)
    tg = torch.randint(1, C, (B,), generator=g)
    lg[:, 0] = 100.0                                          # class 0 never counts, however large its logit
    # planted ranks: R - 1 classes counted ahead of the target (strictly larger, or equal with a lower index), and two equal
    # logits of a higher index that do not count
    b = 0
    for R in (1, 5, 6, 10, 11):
        for t in (1, C - 1, 777):
            row = lg[b]
            others = torch.randperm(C - 2, generator=g) + 1
            others = others[others != t] if t != C - 1 else others
            lower = [int(j) for j in others if j < t][: (R - 1) // 2]
            higher = [int(j) for j in others if j > t][:2]
            rest = [int(j) for j in others if int(j) not in lower and int(j) not in higher][: R - 1 - len(lower)]
            row[t] = 50.0
            row[lower] = 50.0
            row[higher] = 50.0
            row[rest] = 51.0
            tg[b] = t
            b += 1
    skipped = {b: 0, b + 1: C, b + 2: C + 5, b + 3: -1}
    for i, t in skipped.items():
        tg[i] = t
    # exact ranks on the same fp32 logits
    ok = (tg > 0) & (tg < C)
    lt = lg.gather(1, tg.clamp(0, C - 1)[:, None])
    j = torch.arange(C)
    ahead = ((lg > lt) | ((lg == lt) & (j[None, :] < tg[:, None])))[:, 1:].sum(1)
    rank = torch.where(ok, ahead + 1, torch.zeros_like(ahead))
    assert [int(rank[i]) for i in range(15)] == [R for R in (1, 5, 6, 10, 11) for _ in range(3)]
    m0 = torch.tensor([3.0, 4.0, 5.0, 0.5, 0.25, 0.125])
    got, ranks = Fn.eval_rank_metrics(lg.to(_dev()), tg.to(_dev()), metrics=m0.to(_dev()), want_ranks=True)
    got, ranks = got.cpu(), ranks.cpu()
    assert torch.equal(ranks.long(), rank)
    for i, k in enumerate((1, 5, 10)):
        hit = ok & (rank <= k)
        assert got[i].item() == m0[i].item() + int(hit.sum())
        nd = m0[3 + i].item() + (1.0 / torch.log2(rank[hit].double() + 1.0)).sum().item()
        assert abs(got[3 + i].item() - nd) <= 1e-5 * nd, (k, got[3 + i].item(), nd)
