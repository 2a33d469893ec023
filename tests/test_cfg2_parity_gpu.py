"""Parity of the HEADLINE configuration (BASELINE.json configs[1]: HSTU 4 blocks, d=128, h=4, seq_len=200, V=12,101) against the
oracle, plus the training-runtime contracts the advisor asked for (loss scaling in grad-sink mode, dropout seeds across
interleaved forwards, optimizer state)."""
import pytest
import torch

from tests.util import frob_relerr, make_batch, relerr

pytestmark = pytest.mark.gpu

V, L, D, H, NB = 12101, 200, 128, 4, 4


def _cfg2_model(seed=0, dropout=0.0):
    from genrec_b200.hstu import HSTU
    torch.manual_seed(seed)
    m = HSTU(V, L, D, H, NB, dropout=dropout)
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
        if a[3] == f"layers.{NB - 1}.":
            x.retain_grad(); grabbed["x_last"] = x
        return orig(x, *a, **kw)

    oh.hstu_layer_forward = spy
    try:
        if autocast:
            with torch.autocast("cpu", dtype=torch.bfloat16):
                _, lo = oh.hstu_forward(ids, ts, tg, p, H, NB)
            lo.float().backward()
        else:
            _, lo = oh.hstu_forward(ids, ts, tg, p, H, NB)
            lo.backward()
    finally:
        oh.hstu_layer_forward = orig
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    return float(lo), grads, grabbed["x_last"].grad.float()


def test_cfg2_full_model_vs_oracle():
    """Headline configuration, whole model: loss, the gradient entering the last block, the tied embedding-table gradient (through
    the fused V=12,101 CE head with its 95 class tiles and half-block items) and every other parameter gradient, against the fp32
    oracle.  Yardstick = the reference algorithm's OWN bf16-autocast error on the same tensor (north_star's 1e-3 is below what any
    bf16 path, the reference's included, can reach): ours must not exceed it beyond the scatter of the comparison itself.  The table
    is printed (pytest -s)."""
    dev = torch.device("cuda:0")
    B = 8
    m = _cfg2_model()
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    ids, ts, tg = make_batch(B, L, V, seed=5, pad=True)
    ids[3, :57] = 0; ts[3, :57] = 0; tg[3, :56] = 0
    lo, gref, dxref = _oracle_run(ids, ts, tg, sd, autocast=False)
    la, gac, dxac = _oracle_run(ids, ts, tg, sd, autocast=True)
    # ours
    m = m.to(dev).train()
    got = {}

    def grab(mod, args):
        args[0].register_hook(lambda g: got.__setitem__("dx_last", g.clone()))
        return None

    hook = m.layers[NB - 1].register_forward_pre_hook(grab)
    _, loss = m(ids.to(dev), ts.to(dev), tg.to(dev))
    loss.backward()
    hook.remove()
    torch.cuda.synchronize()
    el = abs(loss.item() - lo) / abs(lo)
    ea = abs(la - lo) / abs(lo)
    # (name, ours Frobenius, reference-autocast Frobenius, ours max-norm, reference-autocast max-norm)
    rows = [("loss", el, ea, el, ea),
            ("dX into the last block", frob_relerr(got["dx_last"], dxref), frob_relerr(dxac, dxref), relerr(got["dx_last"], dxref),
             relerr(dxac, dxref))]
    small = set()
    for n, q in m.named_parameters():
        ref = gref[n]
        g = q.grad if q.grad is not None else torch.zeros_like(q)
        if ref.abs().max() == 0:
            assert g.abs().max() == 0, n
            continue
        rows.append((n + ".grad", frob_relerr(g, ref), frob_relerr(gac[n], ref), relerr(g, ref), relerr(gac[n], ref)))
        if ref.numel() < 4096:
            small.add(n + ".grad")
    lines = ["| tensor | ours, Frobenius | reference autocast, Frobenius | ratio | ours, max-norm | reference autocast, max-norm | ratio |",
             "|---|---|---|---|---|---|---|"]
    lines += [f"| {n} | {a:.2e} | {b:.2e} | {a / max(b, 1e-12):.2f} | {c:.2e} | {d:.2e} | {c / max(d, 1e-12):.2f} |" for n, a, b, c, d in rows]
    print("\n".join(lines))
    # Yardstick.  Both columns are one realisation of bf16 rounding noise, so the ratio of the two scatters from tensor to tensor
    # (and, for ours, from build to build: +-10 % on the matrices, a factor ~2 on a 399-entry bias table whose every entry is a
    # cancelling sum of ~10^5 noisy terms).
    #   weight matrices / embedding table / dX (>= 4096 elements): Frobenius error <= 1.1 x the reference algorithm's own
    #       bf16-autocast error, and the geometric mean of the ratio over all of them <= 1.0;
    #   vectors of < 4096 elements (bias tables, norm parameters): <= 3 x each, geometric mean <= 1.25;
    #   the max-norm (one worst element out of up to 1.5 M) is reported and held within 3 x.
    import math
    big_r = [a / b for n, a, b, c, d in rows if n not in small and n != "loss" and b > 0]
    small_r = [a / b for n, a, b, c, d in rows if n in small and b > 0]
    gm = lambda v: math.exp(sum(math.log(max(x, 1e-6)) for x in v) / max(len(v), 1))
    print(f"geometric mean of ours / reference-autocast: matrices {gm(big_r):.3f} ({len(big_r)}), small vectors {gm(small_r):.3f} ({len(small_r)})")
    bad = [(n, a, b, c, d) for n, a, b, c, d in rows if a > (3.0 if n in small else 1.1) * b + 5e-4 or c > 3.0 * d + 1e-3]
    assert not bad, bad
    assert gm(big_r) <= 1.0 and gm(small_r) <= 1.25, (gm(big_r), gm(small_r))
    assert torch.isfinite(m.item_embedding.weight.grad).all()


def test_cfg2_head_logits_vs_oracle():
    from oracle import hstu as oh
    dev = torch.device("cuda:0")
    m = _cfg2_model(seed=2).eval()
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    ids, ts, _ = make_batch(4, L, V, seed=9, pad=True)
    with torch.no_grad():
        ref, _ = oh.hstu_forward(ids, ts, None, sd, H, NB)
        m = m.to(dev)
        logits, _ = m(ids.to(dev), ts.to(dev))
    assert logits.shape == (4, L, V + 1)
    assert relerr(logits, ref) < 2e-2, relerr(logits, ref)
    top = torch.topk(logits[:, -1, 1:].cpu(), 10).indices
    top_ref = torch.topk(ref[:, -1, 1:], 10).indices
    overlap = sum(len(set(a.tolist()) & set(b.tolist())) for a, b in zip(top, top_ref)) / top_ref.numel()
    assert overlap >= 0.9, overlap


@pytest.mark.parametrize("unit", [False])
def test_loss_scaling_reaches_every_gradient_in_sink_mode(unit):
    """FlatAdam grad-sink mode: backward of 0.5 * loss must give 0.5 x every gradient (head and embedding included), and a
    forward that is never back-propagated must leave the flat gradient buffer untouched."""
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatAdam
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    m = HSTU(300, 40, 64, 2, 2, dropout=0.0).to(dev).train()
    opt = FlatAdam(m, lr=1e-3, unit_loss_grad=unit)
    ids, ts, tg = make_batch(6, 40, 300, seed=1, pad=True, device=dev)
    _, loss = m(ids, ts, tg)                    # never back-propagated
    assert opt.grad.abs().max() == 0
    _, loss = m(ids, ts, tg)
    loss.backward()
    g1 = opt.grad.clone()
    opt.grad.zero_()
    _, loss = m(ids, ts, tg)
    (0.5 * loss).backward()
    g2 = opt.grad.clone()
    assert g1.abs().max() > 0
    torch.testing.assert_close(g2, 0.5 * g1, rtol=2e-2, atol=2e-3 * g1.abs().max().item())
    # the head / embedding slots specifically
    o = opt.buffers.offsets[[id(q) for q in opt.params].index(id(m.item_embedding.weight))]
    k = m.item_embedding.weight.numel()
    torch.testing.assert_close(g2[o:o + k], 0.5 * g1[o:o + k], rtol=2e-2, atol=2e-3 * g1[o:o + k].abs().max().item())


def test_unit_loss_grad_fast_path_matches_general_path():
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatAdam
    dev = torch.device("cuda:0")
    ids, ts, tg = make_batch(6, 40, 300, seed=1, pad=True, device=dev)
    grads = []
    for unit in (False, True):
        torch.manual_seed(0)
        m = HSTU(300, 40, 64, 2, 2, dropout=0.0).to(dev).train()
        opt = FlatAdam(m, lr=1e-3, unit_loss_grad=unit)
        _, loss = m(ids, ts, tg)
        loss.backward()
        grads.append(opt.grad.clone())
    torch.testing.assert_close(grads[0], grads[1], rtol=1e-3, atol=1e-4 * grads[0].abs().max().item())


def test_dropout_masks_survive_an_interleaved_forward():
    """Two training forwards before one backward: the backward of the first must re-derive the masks of the FIRST forward (the
    advisor's finding: the device seed counter is bumped by every training forward)."""
    from genrec_b200.hstu import HSTU
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    m = HSTU(300, 40, 64, 2, 2, dropout=0.3).to(dev).train()
    ids, ts, tg = make_batch(6, 40, 300, seed=1, pad=False, device=dev)

    def grads_of(interleave):
        torch.manual_seed(7)
        m._seed_dev = None                                       # same seed stream for both runs
        m.zero_grad(set_to_none=True)
        _, l1 = m(ids, ts, tg)
        if interleave:
            with torch.no_grad():
                m(ids, ts, tg)                                    # bumps the device counter between forward and backward
        l1.backward()
        return l1.item(), {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}

    la, ga = grads_of(False)
    lb, gb = grads_of(True)
    assert abs(la - lb) < 1e-6
    for n in ga:
        torch.testing.assert_close(gb[n], ga[n], rtol=1e-3, atol=1e-5 * max(1.0, ga[n].abs().max().item()))


def test_flat_adam_state_dict_and_mirror_refresh():
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatAdam
    dev = torch.device("cuda:0")
    ids, ts, tg = make_batch(6, 40, 300, seed=1, pad=True, device=dev)

    def make():
        torch.manual_seed(0)
        m = HSTU(300, 40, 64, 2, 2, dropout=0.0).to(dev).train()
        return m, FlatAdam(m, lr=1e-2)

    def step(m, opt):
        _, loss = m(ids, ts, tg)
        loss.backward()
        opt.step()
        return loss.item()

    m1, o1 = make()
    for _ in range(3):
        step(m1, o1)
    ck_model = {k: v.clone() for k, v in m1.state_dict().items()}
    ck_opt = o1.state_dict()
    l_next = step(m1, o1)
    # resume into a fresh model + optimizer: load_state_dict must refresh the bf16 mirror the kernels read
    m2, o2 = make()
    m2.load_state_dict(ck_model)
    o2.load_state_dict(ck_opt)
    assert abs(step(m2, o2) - l_next) < 1e-5
    torch.testing.assert_close(o2.flat, o1.flat, rtol=1e-5, atol=1e-6)
    # manual edit of the masters + explicit refresh
    with torch.no_grad():
        m2.layers[0].ffn[0].weight.data.mul_(0.0)
    o2.refresh_mirror()
    assert o2.mirror_of(m2.layers[0].ffn[0].weight).abs().max() == 0


def test_deferred_weight_gradients_equal_inline_ones():
    """FlatAdam(defer_weight_grads=True): dW / dE GEMMs run on the library's side stream and are joined by step(); gradients and
    the parameter update must equal the inline schedule."""
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatAdam
    import genrec_b200.functional as Fn
    dev = torch.device("cuda:0")
    ids, ts, tg = make_batch(6, 70, 300, seed=1, pad=True, device=dev)
    res = []
    try:
        for defer in (False, True):
            torch.manual_seed(0)
            m = HSTU(300, 70, 64, 2, 2, dropout=0.0).to(dev).train()
            opt = FlatAdam(m, lr=1e-3, unit_loss_grad=True, defer_weight_grads=defer)
            Fn.set_defer_weight_grads(defer)
            gs = []
            for _ in range(2):
                _, loss = m(ids, ts, tg)
                loss.backward()
                opt.sync_grads()
                gs.append(opt.grad.clone())
                opt.step()
            torch.cuda.synchronize()
            res.append((gs, opt.flat.clone()))
    finally:
        Fn.set_defer_weight_grads(False)
        Fn.join_deferred(dev)
    # first step: same kernels, same inputs - only the order of the fp32 reductions (red.global.add) differs between the schedules
    torch.testing.assert_close(res[1][0][0], res[0][0][0], rtol=1e-3, atol=1e-5 * res[0][0][0].abs().max().item())
    # second step: an ulp of difference in a first-step gradient can flip the bf16 rounding of one updated weight in the operand
    # mirror (seen in 3 of 40 repetitions, scripts/flake_deferred.py: 10 elements, 5e-5 of the largest gradient)
    torch.testing.assert_close(res[1][0][1], res[0][0][1], rtol=1e-3, atol=3e-4 * res[0][0][1].abs().max().item())
    assert ((res[1][1] - res[0][1]).abs() > 1e-4).float().mean().item() < 1e-3
