"""TEST INFRASTRUCTURE - COBRA's generate and beam_fusion (genrec/models/cobra.py:531-760) restated from the math with per-user
semantics, for any dtype and device, on tests/cobra_reference.py's encoder and layer pieces.  Each user is decoded alone on its real
items: generated token j sits at position n_b (C+1) + j and attends to the user's n_b (C+1) history rows and its own earlier tokens.
Every step recomputes the whole sequence of every beam (no cache), so this is an independent check of the library's cached path.
Equal totals are ordered by the lower flat index (beam V + token), equal similarities by the lower catalog row, equal fused scores by
the lower beam."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from tests import cobra_reference as cr

# std of the sparse heads' biases in the generation fixtures: wide, so that the beams' totals lead one another by far more than the
# bf16 error of the logits (cobra_params.HEAD_BIAS_STD x GEN_BIAS_SCALE)
GEN_BIAS_SCALE = 100.0
N_ITEMS = 12101                 # catalog of the fusion fixture


def gen_params(P):
    """cobra_params' tensors with the sparse heads' biases spread GEN_BIAS_SCALE times wider"""
    return {k: (v * GEN_BIAS_SCALE if k.startswith("sparse_head.") and k.endswith(".bias") else v) for k, v in P.items()}


def _decoder(P, cfg, h):
    """the decoder stack on unpadded causal sequences h [N, L, D]"""
    H = cfg["decoder_num_heads"]
    pad = torch.zeros(h.shape[:2], dtype=torch.bool, device=h.device)
    for i in range(cfg["decoder_n_layers"]):
        pre = f"decoder.decoder.layers.{i}"
        h = cr._ln(h + cr._mha(h, P, pre + ".self_attn", H, pad, True), P, pre + ".norm1")
        h = cr._ln(h + P[pre + ".multihead_attn.out_proj.bias"].expand_as(h), P, pre + ".norm2")
        h = cr._ln(h + cr._ffn(h, P, pre), P, pre + ".norm3")
    return h


def _top(total, K):
    """the K best of a flat row of totals: descending, equal totals by the lower index"""
    order = torch.sort(total, descending=True, stable=True).indices[:K]
    return total[order], order


def generate_user(P, cfg, ids, text, K, temperature=1.0):
    """one user's n real items: ids [n C], text [n, L] -> (sem_ids [K, C], dense_vecs [K, D], scores [K], leads): leads holds, per
    step, the smallest lead between consecutive selected totals and between the K-th and the (K+1)-th"""
    C, V = cfg.get("n_codebooks", 3), cfg["id_vocab_size"]
    n = text.shape[0]
    dev = text.device
    vecs = cr.encode(P, cfg, text)
    code = ids.view(n, C) + torch.arange(C, device=dev) * V
    Li = n * (C + 1)
    hist = torch.cat([P["cobra_emb.id_embed.weight"][code], vecs.unsqueeze(1)], dim=1).reshape(Li, -1)
    ty = (torch.arange(Li, device=dev) % (C + 1) == C).long()
    hist = hist + P["cobra_emb.pos_embed.weight"][:Li] + P["cobra_emb.type_embed.weight"][ty]
    seqs = torch.zeros(1, 0, dtype=torch.long, device=dev)
    scores = torch.zeros(1, dtype=hist.dtype, device=dev)
    leads = []
    for c in range(C):
        x = hist.unsqueeze(0).expand(seqs.shape[0], -1, -1)
        if c:
            j = torch.arange(c, device=dev)
            gen = P["cobra_emb.id_embed.weight"][seqs + j * V] + P["cobra_emb.pos_embed.weight"][Li + j] + P["cobra_emb.type_embed.weight"][0]
            x = torch.cat([x, gen], dim=1)
        out = _decoder(P, cfg, x)[:, -1]
        logp = F.log_softmax(F.linear(out, P[f"sparse_head.{c}.weight"], P[f"sparse_head.{c}.bias"]) / temperature, dim=-1)
        total = (scores.unsqueeze(-1) + logp).reshape(-1) if c else logp[0]
        top, flat = _top(total, K + 1)
        leads.append(((top[:-1] - top[1:]).min().item()))
        top, flat = top[:K], flat[:K]
        parents, tokens = flat // V, flat % V
        if c == C - 1:
            h_last = out[parents] if c else out.expand(K, -1)
        seqs = torch.cat([seqs[parents], tokens.unsqueeze(-1)], dim=1)
        scores = top
    return seqs, F.normalize(h_last, dim=-1), scores, leads


def real_items(input_ids, C, pad_id):
    return (input_ids.view(input_ids.shape[0], -1, C)[:, :, C - 1] != pad_id).sum(1).tolist()


def generate(P, cfg, input_ids, encoder_input_ids, K, temperature=1.0):
    """-> dict(sem_ids [B, K, C], dense_vecs [B, K, D], scores [B, K], leads [B][C]), each user decoded alone"""
    C = cfg.get("n_codebooks", 3)
    outs = []
    for b, n in enumerate(real_items(input_ids, C, cfg["id_vocab_size"] * C)):
        outs.append(generate_user(P, cfg, input_ids[b, :n * C], encoder_input_ids[b, :n], K, temperature))
    return dict(sem_ids=torch.stack([o[0] for o in outs]), dense_vecs=torch.stack([o[1] for o in outs]),
                scores=torch.stack([o[2] for o in outs]), leads=[o[3] for o in outs])


def best_match(dense, catalog):
    """dense [R, D], catalog [N, D] (unit rows) -> (max similarity [R], its lowest catalog row [R], lead of the best row over the
    runner-up [R])"""
    sim = dense @ catalog.T
    top2 = sim.topk(min(2, sim.shape[1]), dim=-1).values
    mx = top2[:, 0]
    rows = torch.arange(sim.shape[1], device=sim.device)
    best = torch.where(sim == mx[:, None], rows, sim.shape[1]).min(-1).values
    lead = top2[:, 0] - top2[:, 1] if top2.shape[1] > 1 else torch.full_like(mx, float("inf"))
    return mx, best, lead


def beam_fusion(P, cfg, input_ids, encoder_input_ids, item_dense_vecs, item_sem_ids, n_candidates=10, n_beam=50, temperature=1.0,
                alpha=0.5):
    """-> dict(item_ids, sem_ids, scores [B, n_candidates], leads [B, n_candidates]: each rank's fused-score lead over the next
    one (the last rank: over the best unselected beam, inf when none), sim_leads [B, n_candidates]: the similarity lead of each
    rank's catalog row over the beam's runner-up row, gen)"""
    gen = generate(P, cfg, input_ids, encoder_input_ids, n_beam, temperature)
    B = input_ids.shape[0]
    cat = F.normalize(item_dense_vecs.to(gen["dense_vecs"].dtype), dim=-1)
    mx, best, sim_lead = best_match(gen["dense_vecs"].reshape(B * n_beam, -1), cat)
    mx, best, sim_lead = mx.view(B, n_beam), best.view(B, n_beam), sim_lead.view(B, n_beam)
    fused = alpha * torch.softmax(gen["scores"], dim=-1) + (1 - alpha) * ((mx + 1) / 2)
    srt, idx = torch.sort(fused, dim=-1, descending=True, stable=True)
    nxt = torch.cat([srt[:, 1:], torch.full_like(srt[:, :1], float("-inf"))], dim=1)
    item_ids = best.gather(1, idx[:, :n_candidates])
    return dict(item_ids=item_ids, sem_ids=item_sem_ids.to(item_ids.device)[item_ids], scores=srt[:, :n_candidates],
                leads=(srt - nxt)[:, :n_candidates], sim_leads=sim_lead.gather(1, idx[:, :n_candidates]), gen=gen)


def catalog(cfg, dense, seed):
    """[N_ITEMS, d_model] catalog vectors (not unit) and [N_ITEMS, C] semantic ids: random rows, and one row near each row of dense
    [R, d_model] (a user's best beam's dense vector) at seeded places, which every beam of that user then matches by a wide lead"""
    g = torch.Generator().manual_seed(seed)
    D, C, V = cfg["d_model"], cfg["n_codebooks"], cfg["id_vocab_size"]
    vecs = torch.randn(N_ITEMS, D, generator=g)
    rows = torch.randperm(N_ITEMS, generator=g)[:dense.shape[0]]
    vecs[rows] = (dense + 0.3 * torch.randn(dense.shape, generator=g) / D ** 0.5) * (1 + torch.rand(dense.shape[0], 1, generator=g))
    sem = torch.randint(0, V, (N_ITEMS, C), generator=g)
    return vecs, sem
