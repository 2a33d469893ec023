"""genrec_b200.cobra.Cobra.generate / beam_fusion on the GPU: the reference fixture at both shapes, the fp64 restatement
(tests/cobra_generate_reference.py) on a ragged batch and at C = 1 and 2, bit-for-bit invariance of a user's outputs under the batch
around it, the three kernels against fp64 at their edges, and the memory BeamFusion needs for a million-item catalog."""
import math

import pytest
import torch

from tests import cobra_generate_reference as gr
from tests import cobra_params as cp

pytestmark = pytest.mark.gpu
DEV = "cuda"
# score_per_codebook: a score sums one log-probability per codebook, each with the bf16 error of its logits through the decoder
# (measured on an H100 up to 0.020 at C = 1 and 0.031 at C = 3); vec: max-norm relative error of the dense vectors (test_cobra_gpu.py's
# bound); fused: BeamFusion's scores; lead / sim: the fused-score and similarity leads above which a rank's item must match
TOL = dict(score_per_codebook=3e-2, vec=3e-2, fused=1e-2, lead=2e-2, sim=5e-3)


def _rel(a, ref):
    a, ref = a.double().cpu(), ref.double().cpu()
    return ((a - ref).abs().max() / ref.abs().max().clamp_min(1e-300)).item()


def _model(cfg, seed):
    from genrec_b200.cobra import Cobra
    m = Cobra(**cfg)
    m.load_state_dict(gr.gen_params(cp.cobra_params(cp.shapes(cfg), seed)))
    return m.to(DEV)


def _p64(cfg, seed, device=DEV):
    return {k: (v.double() if v.is_floating_point() else v).to(device) for k, v in gr.gen_params(cp.cobra_params(cp.shapes(cfg), seed)).items()}


def _calls(cfg, seed):
    C = cfg["n_codebooks"]
    ids, text = cp.batch(cfg, seed=seed)
    out = [(f"user{b}", ids[b:b + 1, :n * C], text[b:b + 1, :n]) for b, n in enumerate(cp.ITEMS)]
    fids, ftext = cp.batch(cfg, items=(20, 20, 20), seed=seed + 1)
    return out + [("full", fids, ftext)]


def _check_gen(out, ref, users=None):
    users = range(out.sem_ids.shape[0]) if users is None else users
    score_tol = TOL["score_per_codebook"] * out.sem_ids.shape[-1]
    for b in users:
        assert torch.equal(out.sem_ids[b].cpu(), ref["sem_ids"][b].cpu()), b
        assert (out.scores[b].double().cpu() - ref["scores"][b].double().cpu()).abs().max().item() <= score_tol, b
        assert _rel(out.dense_vecs[b], ref["dense_vecs"][b]) <= TOL["vec"], b


@pytest.mark.parametrize("shape", ["small", "trainer"])
def test_generate_and_fusion_match_the_reference_fixture(golden, shape):
    g = golden("cobra_generate.pt")[shape]
    cfg = g["cfg"]
    m = _model(cfg, g["param_seed"])
    for name, ids, text in _calls(cfg, g["batch_seed"]):
        for K in (4, 20):
            _check_gen(m.generate(ids.to(DEV), text.to(DEV), n_candidates=K), g["calls"][f"{name}_k{K}"])
    f = g["fusion"]
    _, fids, ftext = _calls(cfg, g["batch_seed"])[-1]
    vecs, sem = gr.catalog(cfg, g["calls"]["full_k20"]["dense_vecs"][:, 0], f["catalog_seed"])
    out = m.beam_fusion(fids.to(DEV), ftext.to(DEV), vecs.to(DEV), sem.to(DEV), n_candidates=f["n_candidates"], n_beam=f["n_beam"],
                        temperature=f["temperature"], alpha=f["alpha"])
    assert (out.scores.double().cpu() - f["scores"].double()).abs().max().item() <= TOL["fused"]
    lead = f["leads"]
    prev = torch.cat([torch.full_like(lead[:, :1], float("inf")), lead[:, :-1]], dim=1)
    # the rank's beam is settled on both sides, and its catalog row leads the runner-up by more than the bf16 error of a similarity
    sure = (lead > TOL["lead"]) & (prev > TOL["lead"]) & (f["sim_leads"] > TOL["sim"])
    assert bool(sure[:, 0].all())                                    # every user's first rank at least
    assert torch.equal(out.item_ids.cpu()[sure], f["item_ids"][sure])
    assert torch.equal(out.sem_ids.cpu()[sure], f["sem_ids"][sure])


def _settled(ref, margin=TOL["lead"]):
    return [b for b, leads in enumerate(ref["leads"]) if min(leads) > margin]


@pytest.mark.parametrize("C", [1, 2, 3])
def test_generate_matches_the_fp64_restatement_on_a_ragged_batch(C):
    cfg = dict(cp.SMALL, n_codebooks=C)
    m = _model(cfg, 11)
    ids, text = cp.batch(cfg, seed=11)
    for K, T in ((1, 1.0), (7, 0.7), (20, 1.0)):
        ref = gr.generate(_p64(cfg, 11), cfg, ids.to(DEV), text.to(DEV), K, T)
        users = _settled(ref)
        assert len(users) >= 2, ref["leads"]
        _check_gen(m.generate(ids.to(DEV), text.to(DEV), n_candidates=K, temperature=T), ref, users)


def test_a_user_gets_the_same_bits_alone_and_in_any_batch():
    cfg = dict(cp.SMALL)
    C = cfg["n_codebooks"]
    m = _model(cfg, 12)
    ids, text = cp.batch(cfg, seed=12)
    pids, ptext = cp.batch(cfg, seed=12, extra_items=3)              # the same users with three more pad items
    fids, ftext = cp.batch(cfg, items=(20, 20), seed=13)
    for K in (5, 20):
        batch = m.generate(ids.to(DEV), text.to(DEV), n_candidates=K)
        again = m.generate(ids.to(DEV), text.to(DEV), n_candidates=K)
        padded = m.generate(pids.to(DEV), ptext.to(DEV), n_candidates=K)
        for f in batch._fields:
            assert torch.equal(getattr(batch, f), getattr(again, f)), f
            assert torch.equal(getattr(batch, f), getattr(padded, f)), f
        for b, n in enumerate(cp.ITEMS):
            alone = m.generate(ids[b:b + 1, :n * C].to(DEV), text[b:b + 1, :n].to(DEV), n_candidates=K)
            for f in batch._fields:
                assert torch.equal(getattr(batch, f)[b:b + 1], getattr(alone, f)), (b, f)
        # the full-length user of the ragged batch against a batch of full-length users only
        mixed = m.generate(torch.cat([ids[3:4], fids]).to(DEV), torch.cat([text[3:4], ftext]).to(DEV), n_candidates=K)
        full = m.generate(fids.to(DEV), ftext.to(DEV), n_candidates=K)
        for f in batch._fields:
            assert torch.equal(getattr(mixed, f)[0], getattr(batch, f)[3]), f
            assert torch.equal(getattr(mixed, f)[1:], getattr(full, f)), f


def test_generate_keeps_the_training_flag_and_needs_no_gradient():
    m = _model(dict(cp.SMALL, decoder_dropout=0.3), 12).train()
    ids, text = cp.batch(cp.SMALL, seed=12)
    a = m.generate(ids.to(DEV), text.to(DEV), n_candidates=4)
    b = m.generate(ids.to(DEV), text.to(DEV), n_candidates=4)
    assert m.training and not a.scores.requires_grad
    assert torch.equal(a.sem_ids, b.sem_ids) and torch.equal(a.dense_vecs, b.dense_vecs)


# ------------------------------------------------------------------------------------------------ kernel stages
def _bf(t):
    return t.to(torch.bfloat16)


@pytest.mark.parametrize("dh", [32, 64])
@pytest.mark.parametrize("hist", [1, 4, 63, 64, 65, 1021])
def test_beam_attention_stage(dh, hist):
    import genrec_b200.functional as Fn
    g = torch.Generator().manual_seed(hist * 7 + dh)
    H, B = 2, 3
    D = H * dh
    lens = torch.tensor([hist, max(1, hist // 2), 1], dtype=torch.int32)
    for K in (1, 20, 63, 64, 65, 256):
        for S in (1, 2):
            hq = _bf(torch.randn(B, hist, 3 * D, generator=g))
            suf = _bf(torch.randn(S, B * K, 3 * D, generator=g))
            anc = torch.randint(0, B * K, (B * K, S - 1), generator=g, dtype=torch.int32)
            q = suf[S - 1][:, :D]
            out = Fn.cobra_beam_attention(q.to(DEV), hq.to(DEV), lens.to(DEV), suf.to(DEV), anc.to(DEV) if S > 1 else None, S, H)
            # fp64 on the bf16 operands
            ref = torch.empty(B * K, D, dtype=torch.float64)
            for r in range(B * K):
                b = r // K
                ks = [hq[b, :lens[b], D:2 * D]] + [suf[s, anc[r, s], D:2 * D][None] for s in range(S - 1)] + [suf[S - 1, r, D:2 * D][None]]
                vs = [hq[b, :lens[b], 2 * D:]] + [suf[s, anc[r, s], 2 * D:][None] for s in range(S - 1)] + [suf[S - 1, r, 2 * D:][None]]
                kk, vv = torch.cat(ks).double().view(-1, H, dh), torch.cat(vs).double().view(-1, H, dh)
                qq = q[r].double().view(H, dh)
                p = torch.softmax(torch.einsum("hd,jhd->hj", qq, kk) / math.sqrt(dh), dim=-1)
                ref[r] = torch.einsum("hj,jhd->hd", p, vv).reshape(-1)
            err = (out.double().cpu() - ref).abs().max().item()
            assert err <= 1e-2 * ref.abs().max().item() + 1e-3, (K, S, err)


def _topk_check(logits, scores_in, B, K, T, tokens, scores, parents, anc_in=None, anc_out=None):
    """picks against fp64 totals: right values, the order (score desc, flat asc), and no unpicked total above the K-th"""
    V = logits.shape[1]
    K_in = logits.shape[0] // B
    lp = torch.log_softmax(logits.double() / T, dim=-1).view(B, K_in, V)
    tot = (lp + (scores_in.double().view(B, K_in, 1) if scores_in is not None else 0)).view(B, -1)
    flat = (parents * V + tokens).cpu()
    picked = tot.gather(1, flat)
    assert (picked - scores.double().cpu()).abs().max().item() <= 1e-4
    s = scores.cpu()
    assert bool(((s[:, :-1] > s[:, 1:]) | ((s[:, :-1] == s[:, 1:]) & (flat[:, :-1] < flat[:, 1:]))).all())
    rest = tot.scatter(1, flat, float("-inf"))
    assert bool((picked[:, -1] >= rest.max(1).values - 1e-4).all())
    if anc_out is not None:
        rows = (torch.arange(B)[:, None] * K_in + parents.cpu()).reshape(-1)
        exp = torch.cat([anc_in.cpu()[rows] if anc_in is not None else torch.zeros(B * K, 0, dtype=torch.int32), rows[:, None].int()], 1)
        assert torch.equal(anc_out.cpu(), exp)


@pytest.mark.parametrize("V,K", [(256, 1), (256, 20), (64, 64), (512, 512)])
def test_beam_topk_stage(V, K):
    import genrec_b200.functional as Fn
    g = torch.Generator().manual_seed(V + K)
    B = 3
    for K_in in (1, K):
        for T in (1.0, 0.7):
            logits = torch.randn(B * K_in, V, generator=g) * 3
            scores_in = torch.randn(B, K_in, generator=g) if K_in > 1 else None
            anc_in = torch.randint(0, 99, (B * K_in, 2), generator=g, dtype=torch.int32) if K_in > 1 else None
            out = Fn.cobra_beam_topk(logits.to(DEV), scores_in.to(DEV) if scores_in is not None else None, B, K, T,
                                     anc_in.to(DEV) if anc_in is not None else None)
            _topk_check(logits, scores_in, B, K, T, *out[:3], anc_in, out[3])


def test_beam_topk_orders_equal_totals_by_index_and_handles_inf():
    import genrec_b200.functional as Fn
    B, K, V = 2, 20, 64
    logits = torch.zeros(B * K, V)                                  # every total equal: the lowest flat indices, in order
    tokens, scores, parents, _ = Fn.cobra_beam_topk(logits.to(DEV), torch.zeros(B, K, device=DEV), B, K, 1.0)
    flat = (parents * V + tokens).cpu()
    assert torch.equal(flat, torch.arange(K).expand(B, K))
    logits = torch.randn(B * K, V)
    logits[:, ::2] = float("-inf")                                  # half the tokens masked: never picked while others remain
    tokens, scores, parents, _ = Fn.cobra_beam_topk(logits.to(DEV), torch.zeros(B, K, device=DEV), B, K, 1.0)
    assert bool((tokens % 2 == 1).all()) and bool(torch.isfinite(scores).all())
    _topk_check(logits, torch.zeros(B, K), B, K, 1.0, tokens, scores, parents)
    row = torch.randn(1, V)
    row[0, 5] = float("inf")                                        # torch's log_softmax gives NaN: NaN ranks above every number
    tokens, scores, _, _ = Fn.cobra_beam_topk(row.to(DEV), None, 1, 4, 1.0)
    ref = torch.log_softmax(row, dim=-1)[0]
    key = torch.where(torch.isnan(ref), torch.full_like(ref, float("inf")), ref)
    order = torch.sort(key, descending=True, stable=True).indices[:4]
    assert torch.equal(tokens[0].cpu(), order)


@pytest.mark.parametrize("D", [64, 128, 192, 256, 384, 768])
def test_dense_match_stage(D):
    import genrec_b200.functional as Fn
    g = torch.Generator().manual_seed(D)
    for N in (1, 127, 128, 129, 12101):
        R = 200
        table = _bf(torch.randn(N, D, generator=g) / D ** 0.5)
        x = _bf(torch.randn(R, D, generator=g) / D ** 0.5)
        if N > 8:                                                   # planted exact ties: rows 0..3 duplicated at N-4..N-1
            table[N - 4:] = table[:4]
            x[:8] = table[torch.tensor([0, 1, 2, 3, 0, 1, 2, 3])] * 2
        best, item = Fn.cobra_dense_match(x.to(DEV), table.to(DEV))
        sim = x.double() @ table.double().T
        top2 = sim.topk(min(2, N), dim=-1).values
        rows = torch.arange(N)
        ref = torch.where(sim == top2[:, :1], rows, N).min(-1).values
        near = (top2[:, 0] - top2[:, -1] <= 1e-5) if N > 1 else torch.zeros(R, dtype=torch.bool)
        if N > 8:
            assert torch.equal(item.cpu()[:8], torch.tensor([0, 1, 2, 3, 0, 1, 2, 3]))
            near[:8] = False
        assert torch.equal(item.cpu()[~near], ref[~near]), N
        assert (best.double().cpu() - sim.gather(1, item.cpu()[:, None])[:, 0]).abs().max().item() <= 1e-5


def test_beam_fusion_never_forms_the_similarity_matrix():
    """B = 256 users, n_beam 20, a million-item catalog at d_model 384: the reference's [B, n_beam, N] fp32 similarity would be
    20.5 GB; the peak allocation growth of the call stays below a tenth of that"""
    cfg = dict(cp.SMALL, d_model=384, decoder_num_heads=6)
    m = _model(cfg, 14)
    B, N, n_beam = 256, 1_000_000, 20
    ids, text = cp.batch(cfg, items=(20,) * B, text_lens=(3, 8), L=8, seed=14)
    g = torch.Generator(device=DEV).manual_seed(14)
    vecs = torch.randn(N, 384, device=DEV, generator=g)
    sem = torch.randint(0, 256, (N, 3), device=DEV, generator=g)
    ids, text = ids.to(DEV), text.to(DEV)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = m.beam_fusion(ids, text, vecs, sem, n_candidates=10, n_beam=n_beam)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base
    assert growth < B * n_beam * N * 4 / 10, growth
    assert out.item_ids.shape == (B, 10) and bool((out.item_ids >= 0).all()) and bool((out.item_ids < N).all())
