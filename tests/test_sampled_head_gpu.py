"""The sampled-softmax head on the H100 against the fp64 reference of tests/sampled_head_reference.py, which rounds where the
kernels round: token and negative counts on both sides of the 64-class and 128-token tiles, the benchmark token count, a
million-item catalog, the degenerate batches; then the contracts of the C ABI (gradients accumulate, repeat calls give the same
bits), the modules, FlatAdam and a captured training step, and a short training run on the Markov split of test_recall_gpu.py.
The error measures and tolerances are those of the full head (tests/head_reference.py: TOL, head_errors); `pytest -s` prints the
measured errors of every case."""
import pytest
import torch

from tests.head_cases import _dev, _to_dev
from tests.head_reference import TOL, format_table, head_errors, violations
from tests.sampled_head_reference import make_case, reference

pytestmark = pytest.mark.gpu

EPS = 1e-5
_ROWS = []


@pytest.fixture(scope="module", autouse=True)
def _error_table():
    yield
    if _ROWS:
        keys = list(TOL) + ["ignored dx"]
        print("\n" + format_table("", {k: 0.0 for k in keys})[0] + "\n|" + "---|" * (len(keys) + 1))
        print("\n".join(line for _, line in _ROWS))
        print(format_table("max over all cases", {k: max(e[k] for e, _ in _ROWS) for k in keys})[1])


def _call(c, *, dx=None, dtable=None, dg=None, db=None, loss_only=False):
    """grb_head_sampled_loss_forward_backward through the C ABI; zeroed gradient buffers unless given, a workspace of garbage."""
    from genrec_b200 import _lib
    from genrec_b200._lib import check, ptr, stream_ptr
    lib = _lib.load()
    x, tb = c["x"], c["tb"]
    (T, D), C, N = x.shape, tb.shape[0], c["neg"].numel()
    dev = x.device
    ws = torch.full((lib.grb_head_sampled_workspace_bytes(T, D, N),), 0xA5, dtype=torch.uint8, device=dev)
    if not loss_only:
        dx = torch.empty_like(x) if dx is None else dx
        dtable = torch.zeros(C, D, device=dev) if dtable is None else dtable
        dg = torch.zeros(D, device=dev) if dg is None else dg
        db = torch.zeros(D, device=dev) if db is None else db
    loss = torch.empty((), dtype=torch.float32, device=dev)
    check(lib.grb_head_sampled_loss_forward_backward(ptr(x), ptr(c["ln_g"]), ptr(c["ln_b"]), EPS, ptr(tb), ptr(c["tg"]), ptr(c["neg"]),
                                                     ptr(c["log_q"]), T, D, C, N, ptr(loss), ptr(dx), ptr(dtable), ptr(dg), ptr(db), ptr(ws),
                                                     stream_ptr(dev)))
    torch.cuda.synchronize()
    return {"loss": loss.item(), "dx": dx, "dg": dg, "db": db, "dE": dtable}


def _reference(c):
    from genrec_b200 import functional as Fn
    xf, _, st = Fn.layernorm_fwd(c["x"], c["ln_g"], c["ln_b"], EPS)     # ln_fwd_kernel, as the head launches it: the same bits
    return reference(c["x"], st, xf, c["ln_g"], c["tb"], c["tg"], c["neg"], c["log_q"])


def _check(name, c):
    got = _call(c)
    err = head_errors(got, _reference(c), c["tg"])
    _ROWS.append((err, format_table(name, err)[1]))
    assert not violations(err), (name, violations(err), err)
    return got


TN = [(1, 65), (127, 65), (128, 65), (129, 65), (129, 1), (129, 63), (129, 64), (385, 1000), (385, 4096), (129, 8192)]


@pytest.mark.parametrize("T,N", TN)
@pytest.mark.parametrize("D", (64, 128))
def test_sampled_head_vs_fp64(D, T, N):
    c = _to_dev(make_case(T, D, 12102, N, seed=T * 1009 + N * 7 + D, with_log_q=(T + N + D // 64) % 2 == 0))
    _check(f"D={D} C=12102 T={T} N={N}", c)


@pytest.mark.parametrize("D,N", [(128, 1024), (64, 8192)])
def test_benchmark_token_count_vs_fp64(D, N):
    """T = 128 x 200 tokens over 12,101 items: every target repeats, and so do negatives"""
    _check(f"D={D} C=12102 T=25600 N={N}", _to_dev(make_case(25600, D, 12102, N, seed=N)))


def test_million_item_catalog_vs_fp64():
    _check("D=128 C=1000001 T=1000 N=1000", _to_dev(make_case(1000, 128, 1_000_001, 1000, seed=8)))


def test_small_catalog_many_repeats_vs_fp64():
    """C = 7: every id repeats many times among the negatives and the targets, and most negatives hit some token's target"""
    _check("D=64 C=7 T=385 N=200", _to_dev(make_case(385, 64, 7, 200, seed=9)))


def test_every_token_ignored():
    """the convention of the full head: NaN loss, zero gradients"""
    c = _to_dev(make_case(200, 128, 500, 70, seed=1))
    c["tg"].zero_()
    got = _call(c)
    assert got["loss"] != got["loss"]
    assert all(got[k].abs().max().item() == 0.0 for k in ("dx", "dg", "db", "dE"))


def test_all_negatives_equal_and_tokens_with_nothing_but_hits():
    """every negative is item 3: a token whose target is 3 has no negative left (loss 0 and gradient 0 for it), every other token
    sees N copies of the same class"""
    c = make_case(300, 128, 500, 130, seed=2, hits=False)
    c["neg"][:] = 3
    c["tg"][::3] = 3
    c = _to_dev(c)
    got = _check("all negatives equal", c)
    assert got["dx"][c["tg"] == 3].abs().max().item() == 0.0
    only = dict(c)
    only["tg"] = torch.full_like(c["tg"], 3)
    got = _call(only)
    assert got["loss"] == 0.0
    assert all(got[k].abs().max().item() == 0.0 for k in ("dx", "dg", "db", "dE"))


def test_loss_only_call_matches():
    c = _to_dev(make_case(385, 128, 1203, 200, seed=4))
    assert _call(c, loss_only=True)["loss"] == _call(c)["loss"]


@pytest.mark.parametrize("T,D,N", [(385, 64, 130), (2000, 128, 1024)])
def test_gradients_accumulate_and_repeat_calls_give_the_same_bits(T, D, N):
    c = _to_dev(make_case(T, D, 300, N, seed=11))          # C = 300: heavy repeats among targets and negatives
    fresh, again = _call(c), _call(c)
    for k in ("dx", "dg", "db", "dE"):
        assert torch.equal(fresh[k], again[k]), k
    assert fresh["loss"] == again["loss"]
    g = torch.Generator(device=_dev()).manual_seed(3)
    A = {k: torch.randn(fresh[k].shape, device=_dev(), generator=g) * fresh[k].abs().max() for k in ("dE", "dg", "db")}
    got = _call(c, dx=torch.full_like(c["x"], float("nan")), dtable=A["dE"].clone(), dg=A["dg"].clone(), db=A["db"].clone())
    assert torch.equal(got["dx"], fresh["dx"])
    for k in ("dE", "dg", "db"):
        scale = A[k].abs() + fresh[k].abs()
        assert bool(((got[k] - (A[k] + fresh[k])).abs() <= 4 * 2.0 ** -23 * scale + 1e-30).all()), k


# ------------------------------------------------------------------------------------------------ modules
def _models():
    from genrec_b200.hstu import HSTU
    from genrec_b200.sasrec import SASRec
    torch.manual_seed(0)
    V, L = 500, 24
    return V, L, [("hstu", HSTU(V, L, 64, 2, 2, dropout=0.0).to(_dev()).train()), ("sasrec", SASRec(V, L, 64, 2, 2, dropout=0.0).to(_dev()).train())]


def _batch(V, L, B=16):
    g = torch.Generator().manual_seed(5)
    ids = torch.randint(1, V + 1, (B, L), generator=g)
    ids[:4, :5] = 0
    tg = torch.randint(1, V + 1, (B, L), generator=g)
    tg[:4, :4] = 0
    ts = 1_300_000_000 + torch.cumsum(torch.randint(1, 86400, (B, L), generator=g), 1)
    return ids.to(_dev()), ts.to(_dev()), tg.to(_dev())


def test_modules_with_negatives_match_the_reference_on_their_hidden_states():
    from genrec_b200 import functional as Fn
    from genrec_b200.data import sample_negatives
    V, L, models = _models()
    ids, ts, tg = _batch(V, L)
    probs = torch.rand(V + 1, device=_dev()) + 0.1
    neg, log_q = sample_negatives(V, 100, probs=probs)
    for name, m in models:
        args = (ids, ts) if name == "hstu" else (ids,)
        m.zero_grad(set_to_none=True)
        logits, loss = m(*args, tg, negatives=neg, log_q=log_q)
        assert logits is None
        loss.backward()
        got = {k: p.grad.clone() for k, p in m.named_parameters()}
        # the reference on the final hidden states, pushed back through the encoder by autograd
        m.zero_grad(set_to_none=True)
        x = m.encode(*args)
        x2 = x.detach().reshape(-1, x.shape[-1]).contiguous()
        g_, b_ = m.final_norm.weight.detach(), m.final_norm.bias.detach()
        xf, _, st = Fn.layernorm_fwd(x2, g_, b_, m.final_norm.eps)
        ref = reference(x2, st, xf, g_, Fn.cast_bf16(m.item_embedding.weight), tg.reshape(-1), neg, log_q)
        assert abs(loss.item() - ref["loss"]) <= TOL["loss"] * max(1.0, abs(ref["loss"])), name
        x.backward(ref["bf16"]["dx"].float().view_as(x))
        want = {k: (p.grad.clone() if p.grad is not None else torch.zeros_like(p)) for k, p in m.named_parameters()}
        want["item_embedding.weight"] += ref["bf16"]["dE"].float()
        want["final_norm.weight"] += ref["bf16"]["dg"].float()
        want["final_norm.bias"] += ref["bf16"]["db"].float()
        # the encoder's bf16 backward sees dx differing in the last fp32 bits.  A gradient that is zero in exact arithmetic (a key
        # bias under a softmax) is rounding noise in both runs: every parameter is held to at least 1 % of the largest gradient norm
        floor = 1e-2 * max(w.norm().item() for w in want.values())
        for k in got:
            err = (got[k] - want[k]).norm().item() / max(want[k].norm().item(), floor)
            assert err <= 2e-3, (name, k, err)


def test_modules_without_negatives_are_the_full_head_bit_for_bit():
    from genrec_b200 import functional as Fn
    V, L, models = _models()
    ids, ts, tg = _batch(V, L)
    for name, m in models:
        args = (ids, ts) if name == "hstu" else (ids,)
        m.zero_grad(set_to_none=True)
        logits, loss = m(*args, tg)
        loss.backward()
        got = {k: p.grad.clone() for k, p in m.named_parameters()}
        m.zero_grad(set_to_none=True)
        x = m.encode(*args)
        table = m.item_embedding.weight
        want = Fn.HeadLossFn.apply(x, m.final_norm.weight, m.final_norm.bias, table, Fn.cast_bf16(table), tg, m.final_norm.eps)
        want.backward()
        assert logits is None and torch.equal(loss, want), name
        for k, p in m.named_parameters():
            assert torch.equal(got[k], p.grad), (name, k)


def test_op_matches_the_functional():
    import genrec_b200.ops  # noqa: F401
    c = _to_dev(make_case(385, 128, 1203, 200, seed=4))
    want = _call(c)
    x, g, b, table = (c[k].clone().requires_grad_(True) for k in ("x", "ln_g", "ln_b", "table"))
    loss = torch.ops.genrec_b200.head_sampled_loss(x, g, b, table, c["tg"], c["neg"], c["log_q"], EPS)[0]
    (2 * loss).backward()
    assert loss.item() == want["loss"]
    for t, k in ((x, "dx"), (g, "dg"), (b, "db"), (table, "dE")):
        assert torch.equal(t.grad, 2 * want[k]), k


def test_flat_adam_trains_through_it_and_a_captured_step_follows_rewritten_negatives():
    from genrec_b200.data import sample_negatives
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatAdam
    dev = _dev()
    V, L = 500, 24
    ids, ts, tg = _batch(V, L)
    gen = torch.Generator(device=dev).manual_seed(1)
    draws = [sample_negatives(V, 64, generator=gen)[0] for _ in range(6)]

    def run(captured):
        torch.manual_seed(0)
        m = HSTU(V, L, 64, 2, 2, dropout=0.0).to(dev).train()
        opt = FlatAdam(m, lr=1e-3, unit_loss_grad=True)
        neg = draws[0].clone()

        def step():
            _, loss = m(ids, ts, tg, negatives=neg)
            loss.backward()
            opt.step()
            return loss

        losses = []
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for i in range(3):
                neg.copy_(draws[i])
                losses.append(step().item())
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        if captured:
            graph = torch.cuda.CUDAGraph()
            neg.copy_(draws[3])
            with torch.cuda.graph(graph):
                loss = step()
            for i in range(3, 6):
                neg.copy_(draws[i])
                graph.replay()
                losses.append(loss.item())
        else:
            for i in range(3, 6):
                neg.copy_(draws[i])
                losses.append(step().item())
        return losses, torch.cat([p.detach().reshape(-1) for p in m.parameters()])

    eager, p_eager = run(False)
    graphed, p_graph = run(True)
    assert eager == graphed, (eager, graphed)
    assert torch.equal(p_eager, p_graph)
    assert eager[-1] < eager[0]


def test_training_with_uniform_negatives_learns_the_markov_split():
    """HSTU on the synthetic Markov split of test_recall_gpu.py, 150 steps with 32 uniform negatives per step (of 200 items)."""
    from genrec_b200.data import sample_negatives
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatAdam
    from oracle import hstu as oh
    from tests.hstu_cases import markov_users
    dev = _dev()
    V, L, D, H, NB, B, STEPS = 200, 20, 64, 2, 2, 64, 150
    seqs, stamps = markov_users(512, V, L, seed=0)
    train_ids, train_ts, train_tg = seqs[:, :L - 1].to(dev), stamps[:, :L - 1].to(dev), seqs[:, 1:L].to(dev)
    eval_ids, eval_ts, eval_tg = seqs[:, 1:L], stamps[:, 1:L], seqs[:, L]
    torch.manual_seed(0)
    model = HSTU(V, L, D, H, NB, dropout=0.0).to(dev).train()
    opt = FlatAdam(model, lr=3e-3, betas=(0.9, 0.98), unit_loss_grad=True)
    g = torch.Generator().manual_seed(1)
    gen = torch.Generator(device=dev).manual_seed(2)
    losses = []
    for _ in range(STEPS):
        idx = torch.randperm(512, generator=g)[:B].to(dev)
        neg, _ = sample_negatives(V, 32, generator=gen)
        _, loss = model(train_ids[idx], train_ts[idx], train_tg[idx], negatives=neg)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    model.eval()
    top = model.predict(eval_ids.to(dev), eval_ts.to(dev), top_k=10).cpu()
    rec = oh.recall_ndcg(top, eval_tg)["Recall@10"] / 512
    counts = torch.bincount(seqs[:, :L].reshape(-1), minlength=V + 1)
    pop = torch.topk(counts[1:], 10).indices + 1
    rec_pop = float((eval_tg[:, None] == pop[None, :]).any(1).float().mean())
    first, last = sum(losses[:10]) / 10, sum(losses[-10:]) / 10
    print(f"sampled-softmax training: loss {first:.3f} -> {last:.3f}; Recall@10 {rec:.4f}, popularity baseline {rec_pop:.4f}")
    # measured on an H100 80GB HBM3 (700 W power limit): loss 3.252 -> 1.753, Recall@10 0.4434, popularity baseline 0.0527
    assert last < 0.8 * first, (first, last)
    assert rec > 0.25 and rec > 2 * rec_pop, (rec, rec_pop)
