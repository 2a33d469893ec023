"""The tolerances of test_hstu_bias_configs_gpu.py can fail: the fp64 references of its configurations, restated with wrong bucket
logic, land at least 3 tolerances away from the correct ones.  A kernel with one of these mistakes fails those tests."""
import pytest
import torch

from oracle import hstu as oh
from tests import hstu_cases as G

MARGIN = 3.0
POS_TABLE = "position_bias.relative_attention_bias.weight"


def _pos_rule(kind):
    return G.pos_fixed if kind == "fix" else G.pos_reference


# mutation -> (position rule, time rule) built from the correct ones; "collapse" post-processes the gradient instead
def _rules(mutation, pos_fn):
    if mutation == "sign":           # bucket(j - i) instead of bucket(i - j) (and back, for the reference's table)
        return (lambda d, nb, md: pos_fn(-d, nb, md)), G.time_bucket
    if mutation == "pos_shift":      # every position bucket one higher
        return (lambda d, nb, md: torch.clamp(pos_fn(d, nb, md) + 1, max=nb - 1)), G.time_bucket
    if mutation == "time_shift":     # every time bucket one higher
        return pos_fn, (lambda dt, nt: torch.clamp(oh.temporal_bucket(dt, nt) + 1, max=nt - 1))
    if mutation == "time_clamp":     # clamp at ntime - 2 instead of ntime - 1
        return pos_fn, (lambda dt, nt: oh.temporal_bucket(dt, nt - 1))
    return pos_fn, G.time_bucket


def _collapse(dpos):
    out = torch.zeros_like(dpos)
    out[0] = dpos.sum(0)
    return out


MUTATIONS = ["sign", "pos_shift", "time_shift", "time_clamp", "collapse"]


def _applies(mutation, L, ntime, grads=True, kind="fix"):
    """the mutations that exist for a configuration: time ones need a time table of >= 2 buckets; with L = 1 the only cell is the
    diagonal (delta 0, dt 0), so the sign, the time mutations and the collapse change nothing; the collapse needs gradient outside
    bucket 0 (not the reference's table) and a check that sees gradients"""
    if mutation in ("time_shift", "time_clamp"):
        return isinstance(ntime, int) and ntime >= 2 and L >= 2
    if mutation == "sign":
        return L >= 2
    if mutation == "collapse":
        return grads and L >= 2 and kind == "fix"
    return True


# ---------------------------------------------------------------------------------------------------- 2(b) attention core
CORE_PARAMS = [pytest.param(case, mut, id=f"{G.core_id(case)}-{mut}") for case in G.CORE_CASES for mut in MUTATIONS
               if _applies(mut, case[0], case[4], kind=case[3][0])]


@pytest.mark.parametrize("case,mutation", CORE_PARAMS)
def test_core_tolerances_catch_bucket_mistakes(case, mutation):
    L, D, H, pos, time = case
    c = G.core_case(L, D, H, pos, time, seed=L * 7 + D + H)
    pb, tb = G.cell_buckets(c)
    ref = G.core_reference(c, pb, tb)
    if mutation == "collapse":
        mut = dict(ref, dpos=_collapse(ref["dpos"]))
    else:
        pos_fn, time_fn = _rules(mutation, _pos_rule(pos[0]))
        mpb, mtb = G.cell_buckets(c, pos_fn, time_fn)
        mut = G.core_reference(c, mpb, mtb)
    ex = G.core_excess(mut, ref, pb, tb, D)
    assert max(ex.values()) >= MARGIN, ex


# ---------------------------------------------------------------------------------------------------- 2(d) / 2(f) HSTULayer
def _layer_excess(case, mutation, monkeypatch, seed, grads):
    c = G.layer_case(*case, seed=seed)
    G.patch_oracle(monkeypatch, G.pos_fixed)
    ref = G.oracle_layer(c, with_grad=grads)
    if mutation == "collapse":
        y, dx, g = ref
        g = dict(g)
        g[POS_TABLE] = _collapse(g[POS_TABLE])
        return G.layer_excess(y, dx, g, ref)
    G.patch_oracle(monkeypatch, *_rules(mutation, G.pos_fixed))
    return G.layer_excess(*G.oracle_layer(c, with_grad=grads), ref)


LAYER_PARAMS = [pytest.param(case, mut, id="L{}-npos{}-t{}-{}".format(case[0], case[3], case[5], mut)) for case in G.LAYER_CASES
                for mut in MUTATIONS if _applies(mut, case[0], case[5])]


@pytest.mark.parametrize("case,mutation", LAYER_PARAMS)
def test_layer_tolerances_catch_bucket_mistakes(case, mutation, monkeypatch):
    ex = _layer_excess(case, mutation, monkeypatch, case[0] + case[3], grads=True)
    assert max(ex.values()) >= MARGIN, ex


F32_PARAMS = [pytest.param(case, mut, id="L{}-npos{}-t{}-{}".format(case[0], case[3], case[5], mut)) for case in G.F32_LAYER_CASES
              for mut in MUTATIONS if _applies(mut, case[0], case[5], grads=False)]


@pytest.mark.parametrize("case,mutation", F32_PARAMS)
def test_fp32_layer_tolerance_catches_bucket_mistakes(case, mutation, monkeypatch):
    ex = _layer_excess(case, mutation, monkeypatch, case[0] + 3, grads=False)
    assert ex["y"] * G.LAYER_Y_TOL / G.F32_TOL >= MARGIN, ex        # the fp32 test bounds y by F32_TOL


def test_time_bucket_63_is_reached():
    """The batches' widest row reaches the reference's bucket 63, so clamping at 62 is a visible mistake at 64 buckets too."""
    _, ts, _ = G.batch(7, seed=0)
    assert int(oh.temporal_bucket(ts[3, -1:] - ts[3, :1], 64)) == 63
    from genrec_b200.hstu import time_bucket_thresholds
    thr = time_bucket_thresholds()
    d = int(ts[3, -1] - ts[3, 0])
    assert 62 + int(d >= int(thr[63])) == 63                  # the kernels' rule: e = floor(log2 d) = 62, bucket = e + (d >= thr[e+1])
