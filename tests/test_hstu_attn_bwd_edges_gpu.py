"""The HSTU attention backward (Fn.hstu_attention_bwd) against the fp64 references of tests/hstu_block_reference.py at the tile edges
of one to four key tiles and one past them (L = 257), for both head dims and the four kernel instantiations <HAS_TIME, POS_UNI>;
then run-to-run and graph-replay bit identity of dzp and the bias-table gradients.  Every case has B = 4 with a pad in the middle of
row 0, a left-padded row 1 and a fully padded row 2."""
import pytest
import torch

from tests.exact_check import DEV, Ledger
from tests.hstu_cases import _attn_case, core_case, pos_fixed

pytestmark = pytest.mark.gpu
LEDGER = Ledger("worst error / allowance per quantity of the attention backward (tolerance 1):")
_error_table = LEDGER.fixture()

# (pos, time) of the four kernel instantiations <HAS_TIME, POS_UNI>: "ref" buckets are uniform (bucket 0 on every causal cell)
BIAS = [(("fix", 32, 100), 64), (("ref", 32, 128), 64), (("fix", 64, 80), "notable"), (("ref", 32, 128), "nots")]
CASES = [(L, D, H, pos, time) for L in (63, 64, 65, 192, 193, 255, 256, 257) for D, H in ((128, 4), (128, 2)) for pos, time in BIAS]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"L{c[0]}-dh{c[1] // c[2]}-{c[3][0]}{c[3][1]}-t{c[4]}")
def test_attention_backward_vs_fp64(case):
    L, D, H, pos, time = case
    _attn_case(L, D, H, pos, time, seed=L * 5 + D + H, ledger=LEDGER)


def _operands(L, D, H, seed):
    import genrec_b200.functional as Fn
    from genrec_b200.hstu import _thresholds_on
    c = core_case(L, D, H, ("fix", 32, 100), 64, seed)
    pb = pos_fixed(torch.arange(L), 32, 100)
    meta = Fn.SeqMeta(c["pad"].to(torch.uint8).to(DEV), c["ts"].to(DEV), pb.to(torch.uint8).to(DEV), _thresholds_on(DEV), 64, 32,
                      (False, int(pb[0])))
    return c["P"].to(DEV), c["zp"].to(DEV), c["dO"].to(DEV), meta, c["wpos"].to(DEV), c["wtime"].to(DEV)


@pytest.mark.parametrize("L", [200, 256])
def test_two_calls_bit_identical(L):
    """dQ sums its key tiles in a fixed order and the bias-table gradients keep their ordered cross-CTA sum: same bits every call."""
    import genrec_b200.functional as Fn
    P, zp, dO, meta, wpos, wtime = _operands(L, 128, 4, 11)
    a = Fn.hstu_attention_bwd(P, zp, dO, meta, 4, wpos, wtime, 64)
    b = Fn.hstu_attention_bwd(P, zp, dO, meta, 4, wpos, wtime, 64)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def test_graph_replay_matches_eager():
    import genrec_b200.functional as Fn
    P, zp, dO, meta, wpos, wtime = _operands(200, 128, 4, 12)
    eager = Fn.hstu_attention_bwd(P, zp, dO, meta, 4, wpos, wtime, 64)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        Fn.hstu_attention_bwd(P, zp, dO, meta, 4, wpos, wtime, 64)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = Fn.hstu_attention_bwd(P, zp, dO, meta, 4, wpos, wtime, 64)
    for _ in range(2):
        graph.replay()
    torch.cuda.synchronize()
    for x, y in zip(out, eager):
        assert torch.equal(x, y)
