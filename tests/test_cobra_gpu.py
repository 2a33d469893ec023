"""genrec_b200.cobra.Cobra on the GPU: the reference fixture and the fp64 restatement at dropout 0 (every CobraOutput field and
gradient), zero-tensor cross-attention gradients, an AdamW step, the packing invariances (extra text pads change no bit; pad
items change no real item's vector), the empty dense loss, dropout reproducibility, encode_items and the right-padding refusal."""
import pytest
import torch

from tests import cobra_params as cp
from tests import cobra_reference as cr

pytestmark = pytest.mark.gpu
DEV = "cuda"
# bf16 operands with fp32 accumulation through a 1 + 2 (small) or 1 + 8 layer post-LN stack.  Fields and item vectors: max-norm
# relative error.  Gradients: relative Frobenius error - the ReLU-gated linear1 gradients are ill-conditioned enough that a max-norm
# bound would measure their conditioning (an fp32 torch FFN on the same bf16 inputs misses the fp64 max entry by 19 %).
# Measured worst gradient errors: 0.05 for the encoder alone; 0.05 (small) and 0.07 (trainer) for the step against the restatement;
# 0.12 for the trainer step against the sampled fixture (the encoder's position table, reached through eight decoder layers' input
# gradients).  The bounds are 2x and ~1.6x those.
TOL = dict(loss=2e-2, vec=3e-2, grad=1e-1, step_grad=2e-1)


def _rel(a, ref):
    a, ref = a.double().cpu(), ref.double().cpu()
    return ((a - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()


def _gerr(a, ref):
    a, ref = a.double().cpu(), ref.double().cpu()
    return ((a - ref).norm() / ref.norm().clamp_min(1e-300)).item()


def _model(cfg, seed, **kw):
    from genrec_b200.cobra import Cobra
    m = Cobra(**{**cfg, **kw})
    m.load_state_dict(cp.cobra_params(cp.shapes(cfg), seed))
    return m.to(DEV)


def _zero_dropout(m):
    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.p = 0.0
        if isinstance(mod, torch.nn.MultiheadAttention):
            mod.dropout = 0.0
    return m


def _step(m, ids, text):
    m.zero_grad(set_to_none=True)
    out = m(ids.to(DEV), text.to(DEV))
    out.loss.backward()
    return out, {n: p.grad for n, p in m.named_parameters()}


def _check_fields(out, ref):
    for k in ("loss", "loss_sparse", "loss_dense", "codebook_entropy"):
        assert _rel(getattr(out, k), ref[k]) <= TOL["loss"], (k, getattr(out, k).item(), ref[k].item())
    assert abs(out.vec_cos_sim.item() - ref["vec_cos_sim"].item()) <= TOL["vec"]
    for k in ("acc_correct", "acc_total", "recall_correct", "recall_total"):
        assert getattr(out, k).item() == ref[k].item(), k


FIXTURES = ["cobra_small.pt", "cobra_trainer.pt"]


@pytest.mark.parametrize("name", FIXTURES)
def test_step_matches_the_reference_fixture(golden, name):
    g = golden(name)
    cfg = g["cfg"]
    m = _zero_dropout(_model(cfg, g["param_seed"])).train()
    out, grads = _step(m, *cp.batch(cfg, seed=g["batch_seed"]))
    _check_fields(out, g["fields"])
    errs = {n: _gerr(grads[n], v) for n, v in g["vec_grads"].items()}
    for n, s in g["sampled_grads"].items():
        # the sampled entries' error over the norm a sample of that size has on average (the matrix's Frobenius norm scaled by
        # sqrt(samples / entries)): the full-gradient Frobenius error of the restatement test, estimated from the samples.  The
        # samples' own norm would be the wrong scale where most sampled entries are zero (position rows no text reaches).
        a = grads[n].reshape(-1)[s["pos"].long().to(DEV)].double().cpu()
        scale = s["frob"] * (s["pos"].numel() / grads[n].numel()) ** 0.5
        errs[n] = ((a - s["values"].double()).norm() / scale).item()
        assert abs(grads[n].norm().item() - s["frob"]) <= TOL["step_grad"] * s["frob"], n
    assert set(errs) == {n for n, _ in m.named_parameters()}
    print(name, "worst", max(errs.items(), key=lambda kv: kv[1]))
    assert max(errs.values()) <= TOL["step_grad"], errs


@pytest.mark.parametrize("name", FIXTURES)
def test_step_matches_the_fp64_restatement(golden, name):
    """at the fixtures' seeds, whose head logits lead by margins far above the bf16 error (scripts/make_golden_cobra.py), so the
    integer metrics compare exactly"""
    g = golden(name)
    cfg = g["cfg"]
    m = _zero_dropout(_model(cfg, g["param_seed"])).train()
    ids, text = cp.batch(cfg, seed=g["batch_seed"])
    out, grads = _step(m, ids, text)
    ref, rgrads = cr.step(cp.cobra_params(cp.shapes(cfg), g["param_seed"]), cfg, ids, text, device=DEV)
    _check_fields(out, ref)
    errs = {n: _gerr(grads[n], rgrads[n]) for n in rgrads if rgrads[n].abs().max() > 0}
    print("worst", max(errs.items(), key=lambda kv: kv[1]))
    assert max(errs.values()) <= TOL["step_grad"], errs
    for i in range(cfg["decoder_n_layers"]):                     # the empty memory's weights: zero tensors, not None
        pre = f"decoder.decoder.layers.{i}.multihead_attn."
        for n in ("in_proj_weight", "in_proj_bias", "out_proj.weight"):
            assert grads[pre + n] is not None and not grads[pre + n].any(), pre + n


def test_texts_without_tokens_give_the_encoder_zero_gradients():
    """no text has a token: the reference's encoder parameters (all but proj) get zero tensors through the masked pooling"""
    cfg = cp.SMALL
    m = _zero_dropout(_model(cfg, 23)).train()
    ids, text = cp.batch(cfg, seed=24)
    out, grads = _step(m, ids, torch.zeros_like(text))
    assert torch.isfinite(out.loss)
    for n, g in grads.items():
        if n.startswith("encoder.") and not n.startswith("encoder.proj."):
            assert g is not None and not g.any(), n
    assert grads["encoder.proj.bias"].any()


@pytest.mark.parametrize("cfg", [cp.SMALL, cp.TRAINER], ids=["small", "trainer"])
def test_encoder_gradients_match_the_fp64_restatement(cfg):
    """the item-text encoder alone (packed rows, head dim 96, pooled LayerNorm, proj, L2 norm) under a fixed linear loss"""
    m = _zero_dropout(_model(cfg, 19)).train()
    _, text = cp.batch(cfg, seed=20)
    tokens = text.reshape(-1, text.shape[-1])
    w = torch.randn(tokens.shape[0], cfg["d_model"], generator=torch.Generator().manual_seed(21))
    m.zero_grad(set_to_none=True)
    v = m.encode_items(tokens.to(DEV))
    (v * w.to(DEV)).sum().backward()
    P = {k: t.to(DEV).double().requires_grad_() for k, t in cp.cobra_params(cp.shapes(cfg), 19).items() if k.startswith("encoder.")}
    rv = torch.nn.functional.normalize(cr.encode(P, cfg, tokens.to(DEV)), dim=-1)
    (rv * w.to(DEV).double()).sum().backward()
    assert _rel(v, rv) <= TOL["vec"]
    errs = {n: _gerr(p.grad, P[n].grad) for n, p in m.named_parameters() if n in P and P[n].grad.abs().max() > 0}
    print("encoder worst", max(errs.items(), key=lambda kv: kv[1]))
    assert max(errs.values()) <= TOL["grad"], errs


def test_one_adamw_step_matches_the_restatement():
    cfg = cp.SMALL
    m = _zero_dropout(_model(cfg, 5)).train()
    ids, text = cp.batch(cfg, seed=6)
    _step(m, ids, text)
    opt = torch.optim.AdamW(m.parameters(), lr=1e-2, weight_decay=0.01)
    opt.step()
    P = cp.cobra_params(cp.shapes(cfg), 5)
    _, rgrads = cr.step(P, cfg, ids, text, device=DEV)
    ref = {n: torch.nn.Parameter(P[n].to(DEV).double()) for n in rgrads}
    for n, p in ref.items():
        p.grad = rgrads[n]
    torch.optim.AdamW(ref.values(), lr=1e-2, weight_decay=0.01).step()
    checked = 0
    for n, p in m.named_parameters():
        assert p.grad is not None, n                                   # AdamW skips a parameter whose grad is None
        move, rmove = (p.detach().double() - P[n].to(DEV).double()), (ref[n].detach() - P[n].to(DEV).double())
        rg = rgrads[n].abs()
        if not rg.any():
            assert torch.allclose(move, rmove, atol=1e-7), n          # weight decay alone where the gradient is zero
            continue
        # Adam's first step moves an entry by lr * g / (|g| + eps) plus the decay: where |g| is at least half the largest entry the
        # bf16 gradient has the fp64 one's sign, and the two moves agree to far below lr
        big = rg >= 0.5 * rg.max()
        assert (move - rmove)[big].abs().max().item() <= 1e-3 * 1e-2, n
        checked += int(big.sum())
    assert checked > 0


def test_extra_text_pads_change_no_bit():
    cfg = cp.SMALL
    m = _zero_dropout(_model(cfg, 7)).train()
    ids, text = cp.batch(cfg, seed=8, L=128)
    wide = torch.cat([text, torch.zeros(*text.shape[:2], 40, dtype=text.dtype)], dim=2)
    a, ga = _step(m, ids, text)
    ga = {n: g.clone() for n, g in ga.items()}
    b, gb = _step(m, ids, wide)
    for k in a._fields:
        assert torch.equal(getattr(a, k), getattr(b, k)), k
    for n in ga:
        assert torch.equal(ga[n], gb[n]), n


def test_pad_items_change_no_item_vector_and_hold_the_loss():
    cfg = cp.SMALL
    m = _zero_dropout(_model(cfg, 9)).train()
    ids, text = cp.batch(cfg, seed=10)
    ids2, text2 = cp.batch(cfg, seed=10, extra_items=3)
    C, T = cfg["n_codebooks"], text.shape[1]
    with torch.no_grad():
        keep = (ids != m.pad_id).view(len(ids), -1, C)[:, :, -1].reshape(-1).to(torch.uint8).to(DEV)
        keep2 = (ids2 != m.pad_id).view(len(ids2), -1, C)[:, :, -1].reshape(-1).to(torch.uint8).to(DEV)
        v = m._encode(text.reshape(-1, text.shape[-1]).to(DEV), keep).view(len(ids), T, -1)
        v2 = m._encode(text2.reshape(-1, text2.shape[-1]).to(DEV), keep2).view(len(ids), T + 3, -1)
    real = (ids != m.pad_id).view(len(ids), T, C)[:, :, -1].to(DEV)
    assert torch.equal(v[real], v2[:, :T][real])
    a, _ = _step(m, ids, text)
    b, _ = _step(m, ids2, text2)
    assert _rel(b.loss, a.loss) <= 1e-2


def test_no_second_item_gives_the_nan_dense_loss():
    cfg = cp.SMALL
    m = _zero_dropout(_model(cfg, 11)).train()
    ids, text = cp.batch(cfg, items=(1, 1, 1), seed=12)
    out = m(ids.to(DEV), text.to(DEV))
    assert torch.isnan(out.loss_dense) and torch.isnan(out.loss)
    assert torch.isfinite(out.loss_sparse)


def test_dropout_is_reproducible_per_seed():
    cfg = dict(cp.SMALL, decoder_dropout=0.1)
    m = _model(cfg, 13).train()
    ids, text = cp.batch(cfg, seed=14)
    runs = []
    for seed in (1, 1, 2):
        torch.manual_seed(seed)
        out, g = _step(m, ids, text)
        runs.append((out.loss.clone(), {n: t.clone() for n, t in g.items()}))
    assert torch.isfinite(runs[0][0])
    assert torch.equal(runs[0][0], runs[1][0])
    assert all(torch.equal(runs[0][1][n], runs[1][1][n]) for n in runs[0][1])
    assert not torch.equal(runs[0][0], runs[2][0])


def test_encode_items_equals_generate_itemvec():
    cfg = cp.SMALL
    m = _model(cfg, 15).eval()
    _, text = cp.batch(cfg, seed=16)
    with torch.no_grad():
        a = m.generate_itemvec(text.to(DEV))
        b = m.encode_items(text.reshape(-1, text.shape[-1]).to(DEV)).view_as(a)
        ref = cr.encode(cp.cobra_params(cp.shapes(cfg), 15), cfg, text.reshape(-1, text.shape[-1]))
    assert torch.equal(a, b)
    ref = torch.nn.functional.normalize(ref, dim=-1).view_as(a)
    assert _rel(a.cpu(), ref) <= TOL["vec"]


def _pack_rule(tokens, keep):
    """the packing rule on the host: (lengths, first refused text + 1 or 0)"""
    lens, first_bad = [], 0
    for n, t in enumerate(tokens.tolist()):
        z = t.index(0) if 0 in t else len(t)
        if keep is not None and not keep[n]:
            lens.append(0)
        elif any(t[z:]):
            lens.append(0)
            first_bad = first_bad or n + 1
        else:
            lens.append(z)
    return lens, first_bad


def _text(L, n, gap_at=None):
    t = [0] * L
    t[:n] = range(1, n + 1)
    if gap_at is not None:
        t[gap_at] = 7                      # a non-zero token after the text's first zero
    return t


def _many_texts(N, L, refuse):
    """N texts of seeded lengths 0 .. 40.  The longest text (L tokens) and, with refuse, two refused texts sit at the end of the
    batch (N - 2, N - 3 and N - 1), in a chunk after the first of the offsets scan's 1,024-text chunks once N > 1,027; a text that is
    not right-padded but belongs to a pad item (never read) sits at N // 2"""
    g = torch.Generator().manual_seed(N)
    lens = torch.randint(0, 41, (N,), generator=g).tolist()
    texts = [_text(L, n) for n in lens]
    keep = [1] * N
    texts[N - 2] = _text(L, L)
    texts[N // 2] = _text(L, 3, gap_at=70)
    keep[N // 2] = 0
    if refuse:
        texts[N - 3] = _text(L, 35, gap_at=80)
        texts[N - 1] = _text(L, 5, gap_at=9)
    return texts, keep


PACK_CASES = [(False, None), (True, None)] + [(r, n) for n in (1023, 1024, 1025, 5000, 20000) for r in (False, True)]


@pytest.mark.parametrize("refuse,n_texts", PACK_CASES, ids=[str(r) if n is None else f"N{n}-{r}" for r, n in PACK_CASES])
def test_packing_kernels_follow_the_host_rule(refuse, n_texts):
    """lengths 0, 1, 31, 32, 33, 64 and L; keep = 0 over a text that is not right-padded (not refused: a pad item is never read);
    with refuse, texts whose stray token lies in the first 32-token chunk and past it.  With n_texts, that many texts: the offsets
    scan carries its total over chunks of 1,024 texts, and the length / row kernels loop past their grid at 20,000"""
    from genrec_b200 import functional as Fn
    L = 100
    if n_texts is None:
        texts = [_text(L, n) for n in (0, 1, 31, 32, 33, 64, L)] + [_text(L, 3, gap_at=70), _text(L, 40, gap_at=90)]
        keep = [1] * 7 + [0, 0]
        if refuse:
            texts += [_text(L, 5, gap_at=9), _text(L, 35, gap_at=80), _text(L, 64, gap_at=65)]
            keep += [1, 1, 1]
    else:
        texts, keep = _many_texts(n_texts, L, refuse)
    tokens = torch.tensor(texts, dtype=torch.long)
    lens, first_bad = _pack_rule(tokens, keep)
    offsets, info = Fn.cobra_pack_texts(tokens.to(DEV), torch.tensor(keep, dtype=torch.uint8, device=DEV))
    expect = [0]
    for n in lens:
        expect.append(expect[-1] + n)
    assert offsets.tolist() == expect
    assert info.tolist() == [expect[-1], max(lens), first_bad]
    assert (first_bad > 0) == refuse
    tok, pos = Fn.cobra_text_rows(tokens.to(DEV), offsets, expect[-1])
    assert tok.tolist() == [t for i, n in enumerate(lens) for t in texts[i][:n]]
    assert pos.tolist() == [p for n in lens for p in range(n)]


def test_a_text_that_is_not_right_padded_raises():
    cfg = cp.SMALL
    m = _model(cfg, 17)
    ids, text = cp.batch(cfg, seed=18)
    text[1, 0, 0] = 0                                            # a zero before the text's other tokens
    with pytest.raises(ValueError, match="right-padded"):
        m(ids.to(DEV), text.to(DEV))
