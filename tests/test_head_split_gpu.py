"""The fused cross-entropy head with its sweeps cut into segments: each row tile's class sweep and each class tile's token sweep
run as several units on the persistent kernels, every segment continuing from the running sums the one before it left.  At these
shapes the segment counts are above one on any GPU with more than a few SMs: each segment is one to three 64-wide tiles, and the
last token segment of T = 385 is a partial tile.  Checked against the fp64 reference, and for bit-identical repeats."""
import pytest
import torch

from tests.head_reference import make_case, violations, head_errors
from tests.head_cases import _call, _dev, _reference, _to_dev

pytestmark = pytest.mark.gpu

SHAPES = [(385, 64, 1203), (385, 128, 1203), (129, 128, 129)]


def _splits(T, D, C):
    from genrec_b200 import _lib
    lib = _lib.load()
    return lib.grb_head_splits(T, D, C, 0), lib.grb_head_splits(T, D, C, 1)


@pytest.mark.parametrize("T,D,C", SHAPES)
def test_split_head_vs_fp64(T, D, C):
    rs, ts = _splits(T, D, C)
    assert rs > 1 and ts > 1, (rs, ts)
    c = _to_dev(make_case(T, D, C, seed=T * 31 + C + D))
    err = head_errors(_call(c), _reference(c), c["tg"])
    assert not violations(err), (rs, ts, violations(err), err)


@pytest.mark.parametrize("T,D,C", SHAPES[:2])
def test_split_head_repeats_bit_identical_with_and_without_deferred_weight_gradients(T, D, C):
    from genrec_b200 import _lib
    from genrec_b200._lib import check, stream_ptr
    lib = _lib.load()
    c = _to_dev(make_case(T, D, C, seed=17))
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


def _rule(items, span, sms, cap=8):
    """the smallest s whose items * s CTAs (one per SM) leave at most 1/16 of their rounds idle, else the fullest rounds"""
    fills = []
    for s in range(1, min(cap, span) + 1):
        n = items * s
        slots = -(-n // sms) * sms
        if 16 * n >= 15 * slots:
            return s
        fills.append((n / slots, -s))
    return -max(fills)[1]


def test_benchmark_shape_split_counts_fill_the_rounds():
    """cfg2 (T = 128 x 200, C = 12,102): 200 row tiles swept twice over 190 class tiles; 190 class tiles over 400 token tiles"""
    T, D, C = 25600, 128, 12102
    sms = torch.cuda.get_device_properties(_dev()).multi_processor_count
    assert _splits(T, D, C) == (_rule(2 * 200, 190, sms), _rule(190, 400, sms))
    assert _splits(T, 256, C) == (1, 1)
