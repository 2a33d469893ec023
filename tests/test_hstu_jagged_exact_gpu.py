"""The packed (jagged) HSTU path against fp64 references and against its own promises, on the H100.

- One block through grb_hstu_layer_forward_jagged / _backward_jagged under dropout, every stage checked as
  test_hstu_block_exact_gpu.check_block checks the padded block: the row-wise stages on the T token rows with the masks keyed by
  token row (hstu_block_reference.block_stage_items), the attention per sequence.  The cases sit where a packed batch can go wrong:
  key and query tiles past every sequence's end, T at one pass of the gate kernels' row grid and one row past it, T at the M / K
  tails of the wgmma GEMMs, a batch of idle rows only, and 65,535 sequences (the attention grid's z limit).  Idle rows must give
  O = 0, dQ | dK | dV = 0 and dx = 0, and the weight gradients are the sums over the sequence rows alone.  `pytest -s` prints the
  worst error / allowance of every quantity.
- Device offsets out of contract (offsets[B] past T, offsets[0] > 0): no write past T, and the bits of the clamped batch.
- The model against the oracle on the left-padded batch of the same users, with exact_check's autocast yardstick.
- Bit identity: a full-length packed batch is the padded batch (loss, gradients, one FlatAdam step, under dropout), and a user's
  hidden rows and evaluation rank do not depend on the other users of the batch.
- The sampled-softmax head through forward_jagged against tests/sampled_head_reference.py."""
import copy

import pytest
import torch

from tests import dense_reference as dr
from tests import hstu_block_reference as hr
from tests.exact_check import Ledger, row_pass
from tests.hstu_cases import EDGE_LENGTHS, _users, attention_errors_jagged, run_block_jagged

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
LEDGER = Ledger("worst error / allowance per quantity of the packed block (tolerance 1):")
_error_table = LEDGER.fixture()
_record = LEDGER.record


def check_block_jagged(r, case):
    """Every stage of check_block on a packed block; idle rows hold zero gradients and add nothing to the weight gradients."""
    seq = r["seq"]
    items = hr.block_stage_items(r, seq)
    assert not bool(r["dzp"][~seq].any()), "idle rows of dzp are not zero"
    assert not bool(r["dx"][~seq].any()), "idle rows of dx are not zero"
    worst, excess = attention_errors_jagged(r)
    bad = [_record(case, n, dr.worst(got, ref, allow)) for n, got, ref, allow in items]
    bad += [_record(case, "attn " + n, w) for n, w in worst.items()]
    bad += [_record(case, n, w, 1.0) for n, w in excess.items()]
    bad = [b for b in bad if b]
    assert not bad, (case, bad)


# ------------------------------------------------------------------------------------------------ the block, stage by stage
def _pass_lengths(T):
    """EDGE_LENGTHS and sequences of 200 that leave at least one idle row below T -> (lengths, idle)"""
    lengths = EDGE_LENGTHS + [200] * ((T - sum(EDGE_LENGTHS) - 1) // 200)
    return lengths, T - sum(lengths)


E = sum(EDGE_LENGTHS)              # 777 = 6 * 128 + 9
# (why, lengths, idle, D, H, pos, time, p, layer, seed_dev, max_len); "PASS" / "PASS+1" resolve from the SM count as row_pass() does
JAGGED_STAGED = [
    ("row-keyed masks", EDGE_LENGTHS, 5, 128, 4, ("fix", 32, 100), 64, 0.2, 3, None, None),
    ("row-keyed masks", EDGE_LENGTHS, 5, 64, 2, ("uni", 0), 20, 0.2, 0, 7, None),
    ("row-keyed masks", EDGE_LENGTHS, 5, 256, 8, ("uni", 5), "nots", 0.5, 3, None, None),
    ("row-keyed masks", EDGE_LENGTHS, 5, 64, 1, ("fix", 16, 40), 63, 0.5, 0, 123, None),
    ("tiles past every end", [65, 1, 64, 33, 0, 17, 65, 2], 3, 128, 2, ("fix", 32, 128), 64, 0.2, 0, None, 2048),
    ("tiles past every end", [1, 65, 40], 0, 64, 1, ("uni", 0), 20, 0.5, 3, 9, 2048),
    ("row grid pass", "PASS", None, 64, 2, ("fix", 32, 100), 20, 0.5, 0, None, None),
    ("row grid pass + 1", "PASS+1", None, 128, 4, ("uni", 0), "nots", 0.2, 3, 17, None),
    ("T%128=1", EDGE_LENGTHS + [120], 0, 256, 4, ("uni", 0), 64, 0.2, 0, None, None),
    ("T%128=127", EDGE_LENGTHS + [118], 0, 64, 2, ("fix", 32, 100), 20, 0.5, 3, 5, None),
    ("T%128=1 idle", EDGE_LENGTHS, 120, 128, 2, ("fix", 64, 80), "nots", 0.2, 3, None, None),
    ("T%128=127 idle", EDGE_LENGTHS, 118, 256, 8, ("uni", 0), 63, 0.2, 0, 3, None),
    ("idle rows only", [0] * 5, 100, 64, 2, ("fix", 32, 100), 64, 0.2, 0, None, None),
    ("gridDim.z limit", [1] * 65535, 7, 64, 2, ("uni", 0), 64, 0.2, 0, 11, None),
]


def _resolve(case):
    why, lengths, idle = case[:3]
    if lengths in ("PASS", "PASS+1"):
        lengths, idle = _pass_lengths(row_pass() + (lengths == "PASS+1"))
    return (why, lengths, idle) + tuple(case[3:])


def _jid(case):
    why, lengths, idle, D, H, pos, time, p, layer, sd, ml = case
    n = f"B{len(lengths)}-T{sum(lengths) + idle}" if isinstance(lengths, list) else lengths
    return f"{why}-{n}-D{D}-dh{D // H}-{pos[0]}{pos[1]}-t{time}-p{p}-l{layer}-sd{sd}" + (f"-max{ml}" if ml else "")


@pytest.mark.parametrize("case", JAGGED_STAGED, ids=_jid)
def test_jagged_block_stages_vs_fp64(case):
    case = _resolve(case)
    _, lengths, idle, D, H, pos, time, p, layer, sd, ml = case
    r = run_block_jagged(lengths, D, H, pos, time, idle=idle, p=p, layer=layer, seed_dev=sd, max_len=ml)
    assert r["T"] == sum(lengths) + idle
    check_block_jagged(r, _jid(case))
    if sum(lengths) == 0:
        for n, g in r["grads"].items():
            assert bool(torch.isfinite(g).all()) and not bool(g.any()), f"{n}: a batch without tokens has a gradient"


def test_jagged_edges_are_reached():
    """The T of the cases straddle one pass of the gate kernels' row grid on this device and the 128-row GEMM tiles."""
    ts = {sum(c[1]) + c[2] for c in map(_resolve, JAGGED_STAGED)}
    assert {row_pass(), row_pass() + 1} <= ts
    assert {1, 127} <= {t % 128 for t in ts}
    assert E + 120 in ts and E + 118 in ts and (E + 120) % 128 == 1 and (E + 118) % 128 == 127


# ------------------------------------------------------------------------------------------------ device offsets out of contract
_OFF_CASE = dict(D=128, H=4, pos=("fix", 32, 100), time=64)


def _same_bits(a, b, names):
    diff = [n for n in names if not torch.equal(a[n], b[n])]
    diff += [f"grad {n}" for n in a["grads"] if not torch.equal(a["grads"][n], b["grads"][n])]
    assert not diff, diff


def test_device_offsets_past_T_are_clamped_to_T():
    """offsets[B] = T + 40: the last sequence ends at row T, nothing is written to the 64 rows past T in y / dx (the canary rows of
    the same allocations), and every row below T has the bits of the batch with offsets[B] = T."""
    lengths = [63, 129, 40]
    T = sum(lengths) + 24
    ok = [0, 63, 192, T]
    kw = dict(idle=24, p=0.2, layer=1, max_len=200, canary=64)
    a = run_block_jagged(lengths, *_OFF_CASE.values(), offsets=ok, **kw)
    b = run_block_jagged(lengths, *_OFF_CASE.values(), offsets=ok[:-1] + [T + 40], **kw)
    for r in (a, b):
        assert bool((r["y_canary"] == 7.0).all()) and bool((r["dx_canary"] == 7.0).all()), "a write past row T"
    _same_bits(a, b, ("y", "dx", "O", "x1", "xn", "hact", "dzp", "dO", "dx1"))
    check_block_jagged(a, "offsets[B]=T")


def test_device_offsets_with_leading_rows_treat_them_as_idle():
    """offsets[0] = 3: rows 0-2 are idle (O, dzp and dx zero there, no gradient from them) and every sequence row has the bits of
    the same batch without those rows."""
    lengths = [63, 129, 40]
    kw = dict(idle=5, max_len=200, canary=64)
    a = run_block_jagged(lengths, *_OFF_CASE.values(), **kw)
    b = run_block_jagged(lengths, *_OFF_CASE.values(), lead=3, **kw)
    assert b["off"][0] == 3 and not bool(b["seq"][:3].any())
    assert not bool(b["O"][:3].any()) and not bool(b["dzp"][:3].any()) and not bool(b["dx"][:3].any())
    for n in ("y", "dx", "O", "x1", "xn", "hact", "z1", "dzp", "dO", "dx1", "dz1", "dxn"):
        assert torch.equal(a[n], b[n][3:]), n
    for r in (a, b):
        assert bool((r["y_canary"] == 7.0).all()) and bool((r["dx_canary"] == 7.0).all()), "a write past row T"
    check_block_jagged(b, "offsets[0]=3")


# ------------------------------------------------------------------------------------------------ the model against the oracle
def test_model_vs_oracle_within_the_autocast_yardstick():
    """forward_jagged's loss and every parameter gradient at the cfg2 geometry against the fp32 oracle on the left-padded batch of
    the same users (pad-row targets zeroed; HSTU has no absolute positions, so every real token computes the same there), held to
    test_cfg2_full_model_vs_oracle's yardstick: the reference algorithm's own bf16-autocast error.  The batch has an empty history,
    a history of 1, a full one and 23 idle rows."""
    from genrec_b200.data import collate_jagged, pack_jagged
    from tests.exact_check import autocast_yardstick
    from tests.hstu_cases import CFG2_L as L, CFG2_V as V, _cfg2_model, _oracle_run
    from tests.util import frob_relerr, relerr
    lengths = [57, 0, 200, 1, 130, 199, 64, 2]
    m = _cfg2_model()
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    items, ts, off, tgt, _ = _users(lengths, V, 11)
    pb = collate_jagged(items, off, tgt, L, timestamps=ts, max_len_in_batch=L)
    ids_p = pb["input_ids"].cpu()
    tg_p = torch.where(ids_p == 0, 0, pb["targets"].cpu())
    lo, gref, _ = _oracle_run(ids_p, pb["timestamps"].cpu(), tg_p, sd, autocast=False)
    la, gac, _ = _oracle_run(ids_p, pb["timestamps"].cpu(), tg_p, sd, autocast=True)
    m = m.to(DEV).train()
    pk = pack_jagged(items, off, tgt, L, timestamps=ts, num_tokens=sum(lengths) + 23)
    _, loss = m.forward_jagged(pk["input_ids"], pk["offsets"], pk["max_len"], pk["timestamps"], pk["targets"])
    loss.backward()
    torch.cuda.synchronize()
    el, ea = abs(loss.item() - lo) / abs(lo), abs(la - lo) / abs(lo)
    rows, small = [("loss", el, ea, el, ea)], set()
    for n, q in m.named_parameters():
        ref = gref[n]
        g = q.grad if q.grad is not None else torch.zeros_like(q)
        if ref.abs().max() == 0:
            assert g.abs().max() == 0, n
            continue
        rows.append((n + ".grad", frob_relerr(g, ref), frob_relerr(gac[n], ref), relerr(g, ref), relerr(gac[n], ref)))
        if ref.numel() < 4096:
            small.add(n + ".grad")
    autocast_yardstick(rows, small)


# ------------------------------------------------------------------------------------------------ bit identity
def test_full_length_batch_is_the_padded_batch_bit_for_bit():
    """Every length = max_len, no idle rows, dropout 0.2: the token rows, the dropout row keys and the embedding's grids of the
    packed batch are those of the [B, L] batch, so forward_jagged gives forward's loss, every gradient and FlatAdam's state after
    one step, bit for bit."""
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatAdam
    from tests.util import make_batch
    V, B, L = 500, 6, 70
    torch.manual_seed(0)
    mp = HSTU(V, L, 64, 2, 2, dropout=0.2).to(DEV).train()
    mj = copy.deepcopy(mp)
    ids, ts, tg = make_batch(B, L, V, seed=3, pad=False, device=DEV)
    off = torch.arange(0, B * L + 1, L, device=DEV)
    res = []
    for m, run in ((mp, lambda m: m(ids, ts, tg)), (mj, lambda m: m.forward_jagged(ids.view(-1), off, L, ts.view(-1), tg.view(-1)))):
        opt = FlatAdam(m, lr=1e-3)
        _, loss = run(m)
        loss.backward()
        opt.sync_grads()
        grad = opt.grad.clone()
        opt.step()
        torch.cuda.synchronize()
        res.append((loss.detach(), grad, opt.flat.clone(), opt.m.clone(), opt.v.clone(), opt))
    (lp, gp, fp, m1p, v1p, op), (lj, gj, fj, m1j, v1j, _) = res
    assert torch.equal(lp, lj), (lp.item(), lj.item())
    names = dict(mp.named_parameters())
    diff = [n for n, q in names.items()
            for o in [op.buffers.offsets[[id(t) for t in op.buffers.params].index(id(q))]]
            if not torch.equal(gp[o:o + q.numel()], gj[o:o + q.numel()])]
    assert not diff, f"gradients differ in {diff}"
    assert torch.equal(gp, gj)
    assert torch.equal(fp, fj) and torch.equal(m1p, m1j) and torch.equal(v1p, v1j)


def test_a_users_rows_and_rank_do_not_depend_on_the_batch():
    """Evaluation: one user's rows of encode_jagged and their evaluate_batch_jagged rank are the same bits alone, packed after other
    users, and with idle rows behind.  The forward GEMMs and LayerNorm are row-independent and the attention's tiles start at each
    sequence's first row, so a rank never depends on the batch it is served in."""
    from genrec_b200.data import pack_jagged
    from tests.hstu_cases import _jagged_model
    V, n = 300, 77
    others = [130, 5, 200, 0]
    items, ts, off, tgt, _ = _users(others + [n], V, 21)
    m = _jagged_model(V).eval()
    o = off.tolist()
    u_items, u_ts = items[o[-2]:], ts[o[-2]:]

    def run(it, st, lens, tg, idle):
        offs = torch.zeros(len(lens) + 1, dtype=torch.int64)
        offs[1:] = torch.cumsum(torch.tensor(lens), 0)
        pk = pack_jagged(it, offs.to(DEV), tg, 200, timestamps=st, num_tokens=sum(lens) + idle)
        with torch.no_grad():
            x = m.encode_jagged(pk["input_ids"], pk["offsets"], pk["max_len"], pk["timestamps"])
        _, ranks = m.evaluate_batch_jagged(pk["input_ids"], pk["offsets"], pk["max_len"], pk["timestamps"], tg, want_ranks=True)
        s = sum(lens) - n
        return x[s:s + n], ranks[-1]

    alone = run(u_items, u_ts, [n], tgt[-1:], 0)
    packed = run(items, ts, others + [n], tgt, 0)
    behind = run(u_items, u_ts, [n], tgt[-1:], 40)
    for name, (x, rank) in (("packed after other users", packed), ("with idle rows behind", behind)):
        assert torch.equal(x, alone[0]), name
        assert int(rank) == int(alone[1]), name
    assert int(alone[1]) > 0


# ------------------------------------------------------------------------------------------------ the sampled head
def test_forward_jagged_with_negatives_matches_the_reference_on_its_hidden_states():
    """forward_jagged(negatives=, log_q=) against tests/sampled_head_reference.py on encode_jagged's hidden states, the reference's
    dx pushed back through the packed encoder by autograd (as test_sampled_head_gpu does for the padded model).  Idle rows carry
    target 0 and add nothing."""
    from genrec_b200 import functional as Fn
    from genrec_b200.data import pack_jagged, sample_negatives
    from tests.head_reference import TOL
    from tests.sampled_head_reference import reference
    from tests.hstu_cases import _jagged_model
    V = 500
    items, ts, off, tgt, _ = _users(EDGE_LENGTHS, V, 31)
    pk = pack_jagged(items, off, tgt, 200, timestamps=ts, num_tokens=sum(EDGE_LENGTHS) + 19)
    args = (pk["input_ids"], pk["offsets"], pk["max_len"], pk["timestamps"])
    m = _jagged_model(V)
    probs = torch.rand(V + 1, device=DEV) + 0.1
    neg, log_q = sample_negatives(V, 100, probs=probs)
    logits, loss = m.forward_jagged(*args, pk["targets"], negatives=neg, log_q=log_q)
    assert logits is None
    loss.backward()
    got = {k: (p.grad.clone() if p.grad is not None else torch.zeros_like(p)) for k, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    x = m.encode_jagged(*args)
    x2 = x.detach().contiguous()
    g_, b_ = m.final_norm.weight.detach(), m.final_norm.bias.detach()
    xf, _, st = Fn.layernorm_fwd(x2, g_, b_, m.final_norm.eps)
    ref = reference(x2, st, xf, g_, Fn.cast_bf16(m.item_embedding.weight), pk["targets"], neg, log_q)
    assert abs(loss.item() - ref["loss"]) <= TOL["loss"] * max(1.0, abs(ref["loss"])), (loss.item(), ref["loss"])
    x.backward(ref["bf16"]["dx"].float().view_as(x))
    want = {k: (p.grad.clone() if p.grad is not None else torch.zeros_like(p)) for k, p in m.named_parameters()}
    want["item_embedding.weight"] += ref["bf16"]["dE"].float()
    want["final_norm.weight"] += ref["bf16"]["dg"].float()
    want["final_norm.bias"] += ref["bf16"]["db"].float()
    floor = 1e-2 * max(w.norm().item() for w in want.values())
    errs = {k: (got[k] - want[k]).norm().item() / max(want[k].norm().item(), floor) for k in got}
    assert max(errs.values()) <= 2e-3, errs
