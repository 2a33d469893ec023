"""The HSTU block and the fused Adam step against the fp64 references of tests/hstu_block_reference.py, stage by stage and element by
element, at the tile edges of the attention (L around 64 and 128), the grid edges of the gate kernels (T at and one past one pass
of row_grid, and the benchmark's T = 25,600, which wraps it more than once) and of Adam (n around one grid-stride pass).

One block runs forward and backward through grb_hstu_layer_forward / _backward with a saved blob and a workspace this module owns;
the intermediates are read back through the restated carve order, and every stage is checked on the kernel's own inputs to it.
The workspace regions the backward writes start as NaN, so a region (or a row of it) left unwritten shows.  `pytest -s` prints one
table: for every quantity, the worst ratio of error to allowance and the case where it occurred."""
import ctypes as C

import pytest
import torch

from tests import hstu_block_reference as hr
from tests.exact_check import Ledger, _sms, row_pass
from tests.hstu_cases import CORE_CASES, _attn_case, _params, batch, pos_fixed, table_excess

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
LEDGER = Ledger("worst error / allowance per quantity (tolerance 1):")
_error_table = LEDGER.fixture()
_check = LEDGER.check


def adam_pass():
    """elements one grid-stride pass of adam_step_kernel covers: capped_blocks caps at 16 CTAs of 256 threads per SM"""
    return 16 * _sms() * 256


# ------------------------------------------------------------------------------------------------ one block through the C ABI
def _batch(B, L, seed):
    """ids-free pad / ts of B rows: row b follows row b % 4 of hstu_cases.batch (a pad in the middle, a left-padded
    row, a fully padded row, timestamps spanning more than 2^62)."""
    rows = [batch(L, seed + k) for k in range((B + 3) // 4)]
    ts = torch.cat([r[1] for r in rows])[:B]
    pad = torch.cat([r[2] for r in rows])[:B]
    return ts, pad


def run_block(B, L, D, H, p, layer, seed_dev, pos, time, seed=1, defer=False):
    """Forward and backward of one block.  pos: ("uni", bucket) or ("fix", npos, max_distance); time: buckets, "notable" (timestamps,
    no table) or "nots" (no timestamps).  -> dict of inputs, the kernel's intermediates and gradients."""
    import genrec_b200.functional as Fn
    from genrec_b200 import _lib
    from genrec_b200._lib import HstuDims, HstuLayerGrads, HstuLayerParams, HstuSeq, check, ptr, stream_ptr
    from genrec_b200.hstu import _thresholds_on
    lib = _lib.load()
    T = B * L
    ts, pad = _batch(B, L, seed)
    uniform = pos[0] == "uni"
    npos = 8 if uniform else pos[1]
    pb = torch.full((L,), pos[1]) if uniform else pos_fixed(torch.arange(L), pos[1], pos[2])
    has_time = isinstance(time, int)
    ntime = time if has_time else 0
    meta = Fn.SeqMeta(pad.to(torch.uint8).to(DEV), None if time == "nots" else ts.to(DEV), pb.to(torch.uint8).to(DEV),
                      _thresholds_on(DEV), ntime or 64, npos, (uniform, int(pb[0])))
    prm = _params(D, H, npos, ntime, seed + 7)
    g = torch.Generator().manual_seed(seed + 3)
    x = torch.randn(T, D, generator=g)
    x[::3] += 1000.0 * torch.where(torch.arange(0, T, 3) % 2 == 0, 1.0, -1.0)[:, None]
    dy = torch.randint(-64, 65, (T, D), generator=g).float() / 64          # exact: dyb and (p in {0, 0.5}) db2 are bit for bit
    x, dy = x.to(DEV), dy.to(DEV)
    seed_val = None if seed_dev is None else seed_dev
    sdev = None if seed_dev is None else torch.tensor([seed_dev], dtype=torch.int64, device=DEV)
    dseed = 0x1234_5678_9ABC_DEF0 + layer
    dims = HstuDims(B, L, D, H, npos, ntime, float(p), dseed, ptr(sdev), layer)
    names = ("proj_w", "proj_b", "pos_table", "time_table", "ln1_g", "ln1_b", "ffn1_w", "ffn1_b", "ffn2_w", "ffn2_b", "ln2_g", "ln2_b")
    pstruct = HstuLayerParams(*[ptr(prm[n]) if (n != "time_table" or has_time) else None for n in names])
    grads = {n: torch.zeros(prm[n].shape, dtype=torch.float32, device=DEV) for n in names}
    gstruct = HstuLayerGrads(*[ptr(grads[n]) for n in names])
    seq = meta.struct()
    sl, wl = hr.saved_layout(T, D), hr.work_layout(T, D)
    nsaved, nwork = lib.grb_hstu_layer_saved_bytes(C.byref(dims)), lib.grb_hstu_layer_workspace_bytes(C.byref(dims))
    assert nsaved == sl["bytes"], (nsaved, sl["bytes"])
    assert wl["bytes"] <= nwork, (wl["bytes"], nwork)
    saved = torch.full((nsaved,), 0xFF, dtype=torch.uint8, device=DEV)       # NaN in bf16 and fp32
    ws = torch.zeros(nwork, dtype=torch.uint8, device=DEV)
    ws[:wl["bytes"]] = 0xFF
    y, dx = torch.empty_like(x), torch.empty_like(x)
    st = stream_ptr(DEV)
    check(lib.grb_hstu_layer_forward(C.byref(dims), C.byref(pstruct), C.byref(seq), ptr(x), ptr(y), ptr(saved), st))
    if defer:
        check(lib.grb_set_defer_weight_grads(1))
    try:
        check(lib.grb_hstu_layer_backward(C.byref(dims), C.byref(pstruct), C.byref(seq), ptr(dy), ptr(saved), ptr(dx), C.byref(gstruct),
                                          ptr(ws), st))
        if defer:
            check(lib.grb_join_deferred(st))
    finally:
        if defer:
            check(lib.grb_set_defer_weight_grads(0))
    torch.cuda.synchronize()
    out = {n: hr.view(saved, sl, n) for n in sl if n != "bytes"}
    out.update({n: hr.view(ws, wl, n) for n in wl if n != "bytes"})
    out.update(x=x, y=y, dy=dy, dx=dx, grads=grads, prm=prm, pad=pad, meta=meta, B=B, L=L, D=D, H=H, p=p, layer=layer, T=T,
               seed=hr.effective_seed(dseed, p, seed_val), uniform=uniform, npos=npos, pb0=int(pb[0]), has_time=has_time, ntime=ntime)
    return out


def check_block(r, case):
    D, H = r["D"], r["H"]
    prm, gr = r["prm"], r["grads"]
    items = hr.block_stage_items(r)
    # attention forward / backward on the kernel's P, zp and dO
    B, L = r["B"], r["L"]
    wpos = prm["pos_table"][r["pb0"]:r["pb0"] + 1] if r["uniform"] else prm["pos_table"]
    w, masked, pbc, tbc = hr.cell_bias(r["meta"].bias_index, wpos, prm["time_table"][:r["ntime"]] if r["has_time"] else None,
                                       1 if r["uniform"] else r["npos"], H)
    valid = hr.causal_valid(r["pad"].to(DEV))
    assert torch.equal(masked, ~valid), "bias index masks other cells than causal + key padding"
    P3, zp3 = r["P"].view(B, L, 4 * D), r["zp"].view(B, L, 4 * D)
    at = hr.attention(P3, w, valid, H, zp3, r["dO"].view(B, L, D))
    dzp = r["dzp"].view(B, L, 4 * D)
    items += [("O", r["O"].view(B, L, D), at["O"], at["a_O"]), ("dV", dzp[..., D:2 * D], at["dV"], at["a_dV"]),
              ("dQ", dzp[..., 2 * D:3 * D], at["dQ"], at["a_dQ"]), ("dK", dzp[..., 3 * D:], at["dK"], at["a_dK"])]
    if B > 2:
        assert not bool(r["O"].view(B, L, D)[2].any()), "fully padded row: O != 0"
    rows = torch.full_like(pbc, r["pb0"]) if r["uniform"] else pbc
    ref, mass, count = hr.table_sums(at["dS"], valid, rows[:, None], r["npos"])
    ex = {"dpos": table_excess(gr["pos_table"], ref, mass.cpu(), count.cpu())}
    if r["has_time"]:
        ref, mass, count = hr.table_sums(at["dS"], valid, tbc[:, None], r["ntime"])
        ex["dtime"] = table_excess(gr["time_table"], ref, mass.cpu(), count.cpu())
    else:
        assert not bool(gr["time_table"].any()), "time table gradient without a time term"
    del at, w, masked, pbc, tbc, valid
    for n, v in ex.items():
        LEDGER.record(case, n, v)
    assert max(ex.values()) <= 1.0, (case, ex)
    _check(case, items)


def _pass_plus_one_shape():
    """(B, L) with B L = one row-grid pass + 1, B >= 4 where a divisor allows (else B = 1)"""
    n = row_pass() + 1
    for B in range(4, 64):
        if n % B == 0 and n // B <= 16384:
            return B, n // B
    return 1, n


# (B, L, D, H, p, layer, seed_dev, pos, time); "PASS" / "PASS+1" are resolved from the device's SM count
STAGED = [
    (4, 1, 64, 2, 0.0, 0, None, ("fix", 8, 12), 20),
    (4, 63, 128, 2, 0.2, 3, 7, ("uni", 0), 63),
    (4, 64, 256, 8, 0.5, 0, None, ("fix", 32, 100), 64),
    (4, 65, 64, 1, 0.2, 3, None, ("uni", 5), "notable"),
    (4, 127, 128, 4, 0.5, 0, 123, ("fix", 64, 80), "nots"),
    (4, 128, 256, 4, 0.0, 3, None, ("uni", 0), 20),
    (4, 129, 64, 2, 0.2, 0, 99, ("fix", 16, 40), 64),
    (4, 200, 128, 2, 0.5, 3, None, ("fix", 32, 128), 20),
    (4, 257, 256, 8, 0.2, 0, 5, ("uni", 0), 63),
    (128, 200, 128, 4, 0.2, 3, 11, ("uni", 0), 64),                 # the benchmark's block: T = 25,600
    ("PASS", None, 64, 2, 0.5, 0, None, ("fix", 32, 100), 20),      # T = one pass of row_grid
    ("PASS+1", None, 128, 4, 0.2, 3, 17, ("uni", 0), "nots"),       # one row more
    (2, 2048, 256, 8, 0.2, 0, None, ("fix", 32, 128), 64),          # the cfg3 regime
]


def _resolve(case):
    B, L = case[:2]
    if B == "PASS":
        B, L = 4, row_pass() // 4
    elif B == "PASS+1":
        B, L = _pass_plus_one_shape()
    return (B, L) + tuple(case[2:])


def _sid(case):
    B, L, D, H, p, layer, sd, pos, time = case
    return f"B{B}-L{L}-D{D}-dh{D // H if isinstance(H, int) else H}-p{p}-l{layer}-sd{sd}-{pos[0]}{pos[1]}-t{time}"


@pytest.mark.parametrize("case", STAGED, ids=_sid)
def test_block_stages_vs_fp64(case):
    case = _resolve(case)
    r = run_block(*case)
    check_block(r, _sid(case))


def test_block_stages_deferred_weight_grads():
    """The benchmark's schedule: dW GEMMs and bias column sums on the side stream, joined before anything is read."""
    case = (4, 200, 128, 4, 0.2, 3, 3, ("uni", 0), 64)
    check_block(run_block(*case, defer=True), _sid(case) + "-deferred")


def test_edges_are_reached():
    """The chosen T straddle one pass of the gate kernels' row grid and the Adam n one grid-stride pass, on this device."""
    ts = {_resolve(c)[0] * _resolve(c)[1] for c in STAGED}
    assert row_pass() in ts and row_pass() + 1 in ts
    assert 25600 > 2 * row_pass()                      # the benchmark's T wraps the grid more than once
    n = adam_pass()
    assert {n - 1, n, n + 1} <= set(ADAM_N(n))


# ------------------------------------------------------------------------------------------------ attention, element by element
# hstu_cases.CORE_CASES, the shapes of test_attn_tc_gpu (the reference's uniform buckets), and L = 63, 128, 129
ATTN_CASES = list(CORE_CASES) + [(L, D, H, ("ref", 32, 128), t) for L, D, H, t in
                                 [(1, 64, 2, 64), (7, 128, 4, 64), (64, 128, 4, 64), (128, 128, 4, "nots"), (130, 256, 8, 64),
                                  (200, 128, 4, 64), (257, 64, 2, 64), (300, 128, 2, 64), (520, 128, 4, 64)]] + \
    [(63, 64, 1, ("fix", 32, 100), 20), (128, 128, 2, ("ref", 32, 128), 63), (129, 256, 8, ("fix", 64, 80), "notable")]


@pytest.mark.parametrize("case", ATTN_CASES, ids=lambda c: f"L{c[0]}-dh{c[1] // c[2]}-{c[3][0]}{c[3][1]}-t{c[4]}")
def test_attention_elementwise_vs_fp64(case):
    L, D, H, pos, time = case
    _attn_case(L, D, H, pos, time, seed=L * 7 + D + H, ledger=LEDGER)


# ------------------------------------------------------------------------------------------------ Adam
def ADAM_N(n_pass):
    return [1, 255, 257, n_pass - 1, n_pass, n_pass + 1]


def _cfg2_flat_n():
    """FlatAdam's n for the benchmark's model (12,101 items, L = 200, D = 128, H = 4, 4 blocks)"""
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatBuffers
    return FlatBuffers(HSTU(12101, 200, 128, 4, 4)).n


HYPER = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8)


def _adam_state(n, seed):
    g = torch.Generator().manual_seed(seed)
    p = torch.randn(n, generator=g)
    m = 1e-3 * torch.randn(n, generator=g)
    v = 1e-6 * torch.rand(n, generator=g)
    return p.to(DEV), m.to(DEV), v.to(DEV)


def _grad(n, seed):
    """gradients over five decades (1e-5 .. 1), both signs"""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(n, generator=g) * 10.0 ** -torch.randint(0, 6, (n,), generator=g).float()).to(DEV)


def _adam_tick(p, g, m, v, mirror, state, wd, gs, zg, case):
    """one Fn.adam_step from the current buffers, checked against the fp64 step from the same p, m, v"""
    import genrec_b200.functional as Fn
    p0, g0, m0, v0 = p.clone(), g.clone(), m.clone(), v.clone()
    t = int(state[0].item()) + 1
    Fn.adam_step(p, g, m, v, mirror, state, HYPER["lr"], HYPER["beta1"], HYPER["beta2"], HYPER["eps"], wd, gs, zg)
    torch.cuda.synchronize()
    ref = hr.adam(p0, g0, m0, v0, t, weight_decay=wd, grad_scale=gs, **HYPER)
    assert state[0].item() == t
    _check(case, [("adam p", p, ref["p"], ref["a_p"]), ("adam m", m, ref["m"], ref["a_m"]), ("adam v", v, ref["v"], ref["a_v"]),
                  ("adam bc1", state[1:2], torch.tensor([ref["bc1"]]), torch.tensor([ref["a_bc1"]])),
                  ("adam bc2", state[2:3], torch.tensor([ref["bc2"]]), torch.tensor([ref["a_bc2"]]))])
    if mirror is not None:
        assert torch.equal(mirror, p.bfloat16()), "mirror != RNE(p)"
    if zg:
        assert not bool(g.any()), "gradient not zeroed"
    else:
        assert torch.equal(g, g0), "gradient changed"


@pytest.mark.parametrize("which", range(7))
def test_adam_step_vs_fp64(which):
    """n in {1, 255, 257, one grid-stride pass - 1, +0, +1, the cfg2 model's flat size}; weight decay, grad_scale, zero_grad and the
    mirror cycle through the cases; ticks 1, 2 and up to 10, each checked from the kernel's own previous state."""
    n = (ADAM_N(adam_pass()) + [_cfg2_flat_n()])[which]
    wd, gs, zg, mir = (0.0, 1e-2)[which % 2], (1.0, 0.125)[(which // 2) % 2], which % 3 != 1, which % 4 != 2
    p, m, v = _adam_state(n, which)
    mirror = torch.empty(n, dtype=torch.bfloat16, device=DEV) if mir else None
    state = torch.zeros(4, dtype=torch.float32, device=DEV)
    for k in range(10):
        g = _grad(n, 100 * which + k)
        _adam_tick(p, g, m, v, mirror, state, wd, gs, zg, f"adam n={n} wd={wd} gs={gs} zg={zg} mirror={mir} t={k + 1}")


def test_adam_bias_correction_after_1000_ticks():
    """the fp32 device counter after 999 steps, then step 1000 checked alone against fp64 beta^1000"""
    import genrec_b200.functional as Fn
    n = 257
    p, m, v = _adam_state(n, 5)
    state = torch.zeros(4, dtype=torch.float32, device=DEV)
    scratch = [t.clone() for t in (p, m, v)]
    for _ in range(999):
        Fn.adam_step(scratch[0], torch.zeros(n, device=DEV), scratch[1], scratch[2], None, state, HYPER["lr"], HYPER["beta1"],
                     HYPER["beta2"], HYPER["eps"], 0.0, 1.0, True)
    _adam_tick(p, _grad(n, 6), m, v, torch.empty(n, dtype=torch.bfloat16, device=DEV), state, 1e-2, 0.125, True, "adam t=1000")


def test_adam_graph_replay_matches_eager():
    """a captured Fn.adam_step replayed k times: state[0] == k and the same bits as k eager steps"""
    import genrec_b200.functional as Fn
    n, k = adam_pass() + 1, 5
    p, m, v = _adam_state(n, 9)
    g = _grad(n, 10)
    eager = [t.clone() for t in (p, m, v)] + [torch.empty(n, dtype=torch.bfloat16, device=DEV), torch.zeros(4, device=DEV)]
    for _ in range(k):
        Fn.adam_step(eager[0], g.clone(), eager[1], eager[2], eager[3], eager[4], *HYPER.values(), 1e-2, 0.125, False)
    gb = [t.clone() for t in (p, m, v)] + [torch.empty(n, dtype=torch.bfloat16, device=DEV), torch.zeros(4, device=DEV)]
    gg = g.clone()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                       # warm-up outside the capture, then reset the buffers
        Fn.adam_step(gb[0], gg, gb[1], gb[2], gb[3], gb[4], *HYPER.values(), 1e-2, 0.125, False)
    torch.cuda.current_stream().wait_stream(s)
    for t, src in zip(gb[:3], (p, m, v)):
        t.copy_(src)
    gb[4].zero_()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        Fn.adam_step(gb[0], gg, gb[1], gb[2], gb[3], gb[4], *HYPER.values(), 1e-2, 0.125, False)
    for _ in range(k):
        graph.replay()
    torch.cuda.synchronize()
    assert gb[4][0].item() == k
    for a, b in zip(gb, eager):
        assert torch.equal(a, b)


def test_flat_adam_padding_stays_zero():
    """FlatAdam on a small HSTU: the alignment padding between parameter slots stays exactly 0 in p, m, v, the gradient and the
    mirror through several steps.  One head, so the [32, 1] position tables leave 32 elements of padding in their slots."""
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatAdam
    torch.manual_seed(0)
    model = HSTU(97, 40, 64, 1, 2, dropout=0.2).to(DEV).train()
    opt = FlatAdam(model, lr=1e-2, weight_decay=1e-2)
    b = opt.buffers
    live = torch.zeros(b.n, dtype=torch.bool, device=DEV)
    for q, o in zip(b.params, b.offsets):
        live[o:o + q.numel()] = True
    assert bool((~live).any())
    g = torch.Generator().manual_seed(1)
    for step in range(4):
        ids = torch.randint(1, 98, (4, 40), generator=g)
        ts = 1_300_000_000 + torch.cumsum(torch.randint(1, 10 ** 5, (4, 40), generator=g), 1)
        _, loss = model(ids.to(DEV), ts.to(DEV), torch.randint(1, 98, (4, 40), generator=g).to(DEV))
        loss.backward()
        opt.step()
        torch.cuda.synchronize()
        for name, t in (("p", opt.flat), ("m", opt.m), ("v", opt.v), ("grad", opt.grad), ("mirror", opt.mirror)):
            assert not bool(t[~live].any()), (step, name)
