"""FlatAdam(lazy_table=True) on the H100: the row marks of training forwards, the lazy step against the fp64 restatement of
tests/test_lazy_table_cpu.py, bit-identity with the dense FlatAdam where the two must agree, a training run with the sampled head
checked step by step, gradient accumulation, a captured step, checkpoints in both directions, the constructor's refusals and the
Markov-split training run of test_sampled_head_gpu.py."""
import pytest
import torch

from tests.hstu_block_reference import lazy_adam_reference

pytestmark = pytest.mark.gpu


def _dev():
    return torch.device("cuda:0")


def _model(V, D=64, L=16, H=2, blocks=1, seed=0):
    from genrec_b200.hstu import HSTU
    torch.manual_seed(seed)
    return HSTU(V, L, D, H, blocks, dropout=0.0).to(_dev()).train()


def _batch(V, B, L, gen):
    """left-padded ids with repeats, their timestamps, targets with zeros (pads and a few more)"""
    dev = _dev()
    ids = torch.randint(1, V + 1, (B, L), generator=gen)
    ids[0, :5] = 0
    ids[1, :3] = ids[1, 3]                       # a repeated id
    ts = 1_300_000_000 + torch.cumsum(torch.randint(1, 10 ** 5, (B, L), generator=gen), 1)
    ts[ids == 0] = 0
    tg = torch.randint(1, V + 1, (B, L), generator=gen)
    tg[0, :4] = 0
    tg[2, 7] = 0
    return ids.to(dev), ts.to(dev), tg.to(dev)


def _negatives(V, N, gen):
    """uniform negatives with a repeat and ids the kernels ignore (0, negative, >= C)"""
    neg = torch.randint(1, V + 1, (N,), generator=gen)
    neg[1] = neg[0]
    neg[2], neg[3], neg[4] = 0, -3, V + 1 + 5
    return neg.to(_dev())


def _valid(t, C):
    t = t.reshape(-1).cpu()
    return set(t[(t >= 1) & (t < C)].tolist())


def _table_slot(opt):
    C, D = opt._table_rows, opt._table_dim
    sl = slice(opt._table_off, opt._table_off + C * D)
    return [t[sl].view(C, D) for t in (opt.flat, opt.grad, opt.m, opt.v, opt.mirror)]


def _listed_rows(opt):
    n = int(opt._row_count[0])
    rows = opt._row_list[:n].cpu().tolist()
    assert len(rows) == len(set(rows)), "a row was listed twice"
    return set(rows), n


def test_marks_are_the_rows_the_kernels_can_write_and_the_step_clears_them():
    from genrec_b200.optim import FlatAdam
    V, C = 300, 301
    m = _model(V)
    opt = FlatAdam(m, lr=1e-3, unit_loss_grad=True, lazy_table=True)
    gen = torch.Generator().manual_seed(0)
    want = set()
    losses = []
    for _ in range(2):                                           # marks accumulate over two training forwards
        ids, ts, tg = _batch(V, 4, 16, gen)
        neg = _negatives(V, 40, gen)
        losses.append(m(ids, ts, tg, negatives=neg)[1])
        want |= _valid(ids, C) | _valid(tg, C) | _valid(neg, C)
    extra = torch.tensor([[0, C, C + 17, 5], [-1, 5, 299, 300]], device=_dev())   # ids >= C, pads and repeats, straight to the marker
    opt._mark(extra)
    want |= _valid(extra, C)
    torch.cuda.synchronize()
    got, n = _listed_rows(opt)
    assert got == want and n == len(want)
    flag = opt._row_flag.cpu()
    assert set(torch.nonzero(flag).view(-1).tolist()) == want and int(flag.max()) == 1
    assert 0 not in got and int(opt._row_count[1]) == 0
    with torch.no_grad():                                        # no grad: no marks
        m(*_batch(V, 4, 16, gen)[:2])
    assert _listed_rows(opt)[1] == n
    sum(losses).backward()
    opt.step()
    torch.cuda.synchronize()
    assert int(opt._row_flag.abs().sum()) == 0 and opt._row_count.tolist() == [0, 0]
    assert int(torch.count_nonzero(_table_slot(opt)[1])) == 0
    # a full-head forward asks for every row
    ids, ts, tg = _batch(V, 4, 16, gen)
    m(ids, ts, tg)[1].backward()
    torch.cuda.synchronize()
    assert int(opt._row_count[1]) == 1
    opt.step()
    torch.cuda.synchronize()
    assert opt._row_count.tolist() == [0, 0] and int(opt._row_flag.abs().sum()) == 0


def _rule(opt, step):
    """the optimizer's hyper-parameters as the kernels see them: fp32 betas and the bias corrections its state holds after `step`"""
    f32 = lambda x: float(torch.tensor(x, dtype=torch.float32))  # noqa: E731
    bc = opt.state.cpu()
    assert float(bc[0]) == step
    return dict(lr=opt.lr, betas=(f32(opt.betas[0]), f32(opt.betas[1])), eps=opt.eps, weight_decay=opt.weight_decay,
                bias_corrections=(float(bc[1]), float(bc[2])))


def _dense_params_reference(opt, before, step):
    """fp64 dense rule on every element outside the table slot -> (p, m, v) of those elements"""
    lo, hi = opt._table_off, opt._table_off + opt._table_rows * opt._table_dim
    keep = torch.ones(opt.n, dtype=torch.bool)
    keep[lo:hi] = False
    p, g, m, v = (t[keep][:, None] for t in before[:4])
    return lazy_adam_reference(p, g, m, v, range(p.shape[0]), step, **_rule(opt, step)), keep


def _check_step_against_reference(opt, before, rows, step, *, check_dense=True):
    """`before` = (flat, grad, m, v, mirror) on the CPU before the step; checks the table rows and the rest after it"""
    C, D = opt._table_rows, opt._table_dim
    lo = opt._table_off
    after = [t.detach().cpu() for t in (opt.flat, opt.grad, opt.m, opt.v, opt.mirror)]
    tab = lambda t: t[lo:lo + C * D].view(C, D)  # noqa: E731
    p_ref, m_ref, v_ref = lazy_adam_reference(tab(before[0]), tab(before[1]), tab(before[2]), tab(before[3]), rows, step,
                                              **_rule(opt, step))
    r = sorted(rows)
    untouched = torch.ones(C, dtype=torch.bool)
    untouched[r] = False
    p, g, m, v, mir = (tab(t) for t in after)
    for new, old in zip((p, m, v, mir), (tab(before[0]), tab(before[2]), tab(before[3]), tab(before[4]))):
        assert torch.equal(new[untouched], old[untouched]), "an untouched row changed"
    if r:
        upd_ref = p_ref[r] - tab(before[0])[r].double()
        upd = p[r].double() - tab(before[0])[r].double()
        err = (upd - upd_ref).abs().max().item()
        assert err <= 2e-5 * upd_ref.abs().max().item() + 2 ** -23 * tab(before[0])[r].abs().max().item() * 2, err
        # m can cancel (beta1 m against (1 - beta1) g), and so can g itself against weight_decay p: the errors of both moments are
        # measured against the row set's largest one
        torch.testing.assert_close(m[r].double(), m_ref[r], rtol=2e-6, atol=1e-6 * m_ref[r].abs().max().item())
        torch.testing.assert_close(v[r].double(), v_ref[r], rtol=2e-6, atol=1e-6 * v_ref[r].abs().max().item())
        assert torch.equal(mir[r], p[r].to(torch.bfloat16)), "the mirror is not bf16(p) on a touched row"
    assert int(torch.count_nonzero(g[r])) == 0, "a touched gradient row was not zeroed"
    assert torch.equal(g[untouched], tab(before[1])[untouched]), "an untouched gradient row changed"
    if check_dense:
        (pd, md, _), keep = _dense_params_reference(opt, before, step)
        upd = after[0][keep].double()[:, None] - before[0][keep].double()[:, None]
        upd_ref = pd - before[0][keep].double()[:, None]
        err = (upd - upd_ref).abs().max().item()
        assert err <= 2e-5 * upd_ref.abs().max().item() + 2 ** -23 * before[0][keep].abs().max().item() * 2, err
        torch.testing.assert_close(after[2][keep].double()[:, None], md, rtol=2e-6, atol=1e-6 * md.abs().max().item())


@pytest.mark.parametrize("D,wd", [(64, 0.0), (64, 0.01), (128, 0.0), (128, 0.01), (256, 0.0), (256, 0.01)])
def test_lazy_step_matches_the_fp64_rule(D, wd):
    """seeded gradients in every element (untouched table rows too: the step must leave them and their gradient alone), a different
    row set at every step, one step with no row at all"""
    from genrec_b200.optim import FlatAdam
    V = 1500
    m = _model(V, D=D, H=D // 64 * 2 if D == 256 else 2)
    opt = FlatAdam(m, lr=1e-2, betas=(0.9, 0.99), eps=1e-6, weight_decay=wd, lazy_table=True)
    C = V + 1
    gen = torch.Generator(device=_dev()).manual_seed(D)
    for step in range(1, 8):
        opt.grad.add_(torch.randn(opt.n, device=_dev(), generator=gen))
        if step == 4:
            ids = torch.zeros(0, dtype=torch.int64, device=_dev())            # count 0: only the dense parameters step
        else:
            ids = torch.randint(-5, C + 5, (37 * step,), device=_dev(), generator=gen)
        opt._mark(ids)
        before = [t.detach().cpu() for t in (opt.flat, opt.grad, opt.m, opt.v, opt.mirror)]
        opt.step()
        torch.cuda.synchronize()
        assert float(opt.state[0]) == step
        _check_step_against_reference(opt, before, _valid(ids, C), step)


def _train(lazy, batches, *, V=200, unit=True, wd=0.0):
    from genrec_b200.optim import FlatAdam
    m = _model(V)
    opt = FlatAdam(m, lr=3e-3, weight_decay=wd, unit_loss_grad=unit, lazy_table=lazy)
    for ids, ts, tg, neg in batches:
        _, loss = m(ids, ts, tg, negatives=neg)
        loss.backward()
        opt.step()
    torch.cuda.synchronize()
    return m, opt


def test_full_head_is_bit_identical_to_dense():
    gen = torch.Generator().manual_seed(3)
    batches = [(*_batch(200, 4, 16, gen), None) for _ in range(4)]
    for wd in (0.0, 0.01):
        (md, od), (ml, ol) = _train(False, batches, wd=wd), _train(True, batches, wd=wd)
        for a, b in zip(md.parameters(), ml.parameters()):
            assert torch.equal(a, b)
        for name in ("flat", "m", "v", "mirror", "state"):
            assert torch.equal(getattr(od, name), getattr(ol, name)), name


def test_rows_touched_at_every_step_follow_dense_bit_for_bit():
    """the same batch and negatives every step: every row the forward reads is touched at every step (and, at weight_decay 0, the
    dense step leaves the never-touched rows alone), so the sampled-head run is the dense run"""
    gen = torch.Generator().manual_seed(4)
    ids, ts, tg = _batch(200, 4, 16, gen)
    neg = _negatives(200, 48, gen)
    batches = [(ids, ts, tg, neg)] * 5
    (md, od), (ml, ol) = _train(False, batches), _train(True, batches)
    for a, b in zip(md.parameters(), ml.parameters()):
        assert torch.equal(a, b)
    assert torch.equal(od.m, ol.m) and torch.equal(od.v, ol.v) and torch.equal(od.mirror, ol.mirror)


def _run_checked(passes, steps=4, unit=True):
    """HSTU with the sampled head; before each step the flat gradient is read and the fp64 rule applied on the CPU set of touched
    rows, after it the step is compared: touched rows within rounding, every other row unchanged, the gradient slot zero"""
    from genrec_b200.optim import FlatAdam
    V, C = 400, 401
    m = _model(V)
    opt = FlatAdam(m, lr=3e-3, unit_loss_grad=unit, lazy_table=True)
    gen = torch.Generator().manual_seed(5 + passes)
    for step in range(1, steps + 1):
        touched = set()
        for _ in range(passes):
            ids, ts, tg = _batch(V, 4, 16, gen)
            neg = _negatives(V, 32, gen)
            _, loss = m(ids, ts, tg, negatives=neg)
            loss.backward()
            touched |= _valid(ids, C) | _valid(tg, C) | _valid(neg, C)
        opt.sync_grads()
        torch.cuda.synchronize()
        assert _listed_rows(opt)[0] == touched
        before = [t.detach().cpu() for t in (opt.flat, opt.grad, opt.m, opt.v, opt.mirror)]
        opt.step()
        torch.cuda.synchronize()
        _check_step_against_reference(opt, before, touched, step)
        p_old, g_old, m_old = _table_slot_of(before[:3], opt)
        changed = set(torch.nonzero((p_old != _table_slot(opt)[0].cpu()).any(1)).view(-1).tolist())
        # a touched row stays put only when its gradient and momentum are both zero (a target whose token is a pad: h = LN(0) = 0
        # at initialisation)
        moving = set(torch.nonzero((g_old != 0).any(1) | (m_old != 0).any(1)).view(-1).tolist()) & touched
        assert changed == moving and len(moving) >= 0.9 * len(touched), (len(changed), len(moving), len(touched))
        assert int(torch.count_nonzero(_table_slot(opt)[1])) == 0


def _table_slot_of(ts, opt):
    C, D = opt._table_rows, opt._table_dim
    return [t[opt._table_off:opt._table_off + C * D].view(C, D) for t in ts]


def test_sampled_head_training_matches_the_rule_step_by_step():
    _run_checked(passes=1)


def test_gradient_accumulation_steps_the_union_of_the_row_sets():
    _run_checked(passes=2, steps=3)
    _run_checked(passes=2, steps=2, unit=False)


def test_a_captured_step_follows_rewritten_ids_targets_and_negatives():
    from genrec_b200.optim import FlatAdam
    V, B, L = 500, 4, 16
    gen = torch.Generator().manual_seed(6)
    draws = [(*_batch(V, B, L, gen), _negatives(V, 64, gen)) for _ in range(6)]

    def run(captured):
        m = _model(V)
        opt = FlatAdam(m, lr=1e-3, unit_loss_grad=True, lazy_table=True)
        ids, ts, tg, neg = (t.clone() for t in draws[0])

        def load(i):
            for dst, src in zip((ids, ts, tg, neg), draws[i]):
                dst.copy_(src)

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
                load(i)
                losses.append(step().item())
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        if captured:
            graph = torch.cuda.CUDAGraph()
            load(3)
            with torch.cuda.graph(graph):
                loss = step()
            for i in range(3, 6):
                load(i)
                graph.replay()
                losses.append(loss.item())
        else:
            for i in range(3, 6):
                load(i)
                losses.append(step().item())
        return losses, torch.cat([opt.flat, opt.m, opt.v]), opt._row_count.tolist()

    eager, s_eager, _ = run(False)
    graphed, s_graph, counts = run(True)
    again, s_again, _ = run(True)
    assert eager == graphed == again, (eager, graphed, again)
    assert torch.equal(s_eager, s_graph) and torch.equal(s_graph, s_again)
    assert counts == [0, 0]
    assert eager[-1] < eager[0]


def test_checkpoints_move_between_dense_and_lazy():
    from genrec_b200.optim import FlatAdam
    V = 200
    gen = torch.Generator().manual_seed(7)
    sampled = [(*_batch(V, 4, 16, gen), _negatives(V, 32, gen)) for _ in range(3)]
    full = (*_batch(V, 4, 16, gen), None)
    m1, lazy = _train(True, sampled, V=V)
    sd, msd = lazy.state_dict(), {k: v.clone() for k, v in m1.state_dict().items()}
    assert sd["n"] == lazy.n and set(sd) == {"m", "v", "state", "hyper", "n"}
    m2 = _model(V, seed=1)
    dense = FlatAdam(m2, lr=3e-3, unit_loss_grad=True)
    m2.load_state_dict(msd)
    dense.load_state_dict(sd)
    assert dense.n == lazy.n
    for name in ("flat", "m", "v", "mirror", "state"):
        assert torch.equal(getattr(dense, name), getattr(lazy, name)), name
    # one more step with the full head on both: it touches every row, so both optimizers compute the same bits
    for mod, opt in ((m1, lazy), (m2, dense)):
        mod(*full[:3])[1].backward()
        opt.step()
    torch.cuda.synchronize()
    for name in ("flat", "m", "v", "state"):
        assert torch.equal(getattr(dense, name), getattr(lazy, name)), name
    # and back: the dense state into a fresh lazy optimizer, which trains on
    m3 = _model(V, seed=2)
    lazy2 = FlatAdam(m3, lr=3e-3, unit_loss_grad=True, lazy_table=True)
    m3.load_state_dict(m2.state_dict())
    lazy2.load_state_dict(dense.state_dict())
    assert torch.equal(lazy2.m, dense.m) and torch.equal(lazy2.mirror, dense.mirror)
    for mod, opt in ((m2, dense), (m3, lazy2)):
        ids, ts, tg, neg = sampled[0]
        loss = mod(ids, ts, tg, negatives=neg)[1]
        loss.backward()
        opt.step()
        assert torch.isfinite(loss).item()
    torch.cuda.synchronize()
    assert float(lazy2.state[0]) == 5.0


def test_constructor_refusals_on_the_gpu():
    from genrec_b200.optim import FlatAdam
    with pytest.raises(ValueError, match="exactly one HSTU"):
        FlatAdam(torch.nn.Linear(8, 8).to(_dev()), lazy_table=True)
    with pytest.raises(ValueError, match="exactly one HSTU"):
        FlatAdam(torch.nn.ModuleList([_model(20), _model(20)]), lazy_table=True)
    with pytest.raises(ValueError, match="grad_sink"):
        FlatAdam(_model(20), lazy_table=True, grad_sink=False)


def test_training_with_uniform_negatives_and_lazy_table_learns_the_markov_split():
    """test_sampled_head_gpu.py's Markov run (150 steps, 32 uniform negatives of 200 items) with lazy_table=True"""
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
    opt = FlatAdam(model, lr=3e-3, betas=(0.9, 0.98), unit_loss_grad=True, lazy_table=True)
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
    print(f"sampled-softmax training, lazy_table=True: loss {first:.3f} -> {last:.3f}; Recall@10 {rec:.4f}, "
          f"popularity baseline {rec_pop:.4f}")
    assert last < 0.8 * first, (first, last)
    assert rec > 0.25 and rec > 2 * rec_pop, (rec, rec_pop)
