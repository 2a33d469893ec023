"""Write tests/golden/cobra_generate.pt from the reference's unmodified Cobra.generate and Cobra.beam_fusion (genrec/models/cobra.py:
531-760) on the CPU in fp32, every dropout p set to 0, at the SMALL and at the trainer's shape (tests/cobra_params.py):

    per user   each user of cobra_params.batch (1, 2, 7 and 20 items) alone, input_ids[b:b+1, :n_b C] (the per-user semantics
               genrec_b200.cobra.Cobra.generate implements), n_candidates 4 and 20
    batched    one call on three users of 20 items each (where the reference's batched call already is per user), n_candidates 4, 20
    fusion     beam_fusion on the batched users at the trainer's eval call (n_candidates 10, n_beam 20, alpha 0.5) over a seeded
               catalog of 12,101 items, with a row planted near each user's best beam's dense vector

The parameters are not stored: the tests rebuild them from (shapes, param_seed) with cobra_generate_reference.gen_params.  The
seeds are searched until, at every step of every call, the consecutive selected totals and the K-th against the (K+1)-th lead by at
least MARGIN (measured on the fp64 restatement of tests/cobra_generate_reference.py), so the beams of a bf16 model can be compared
exactly.  The fused scores' per-rank leads, and each rank's similarity lead of its catalog row over the runner-up, are stored
with the fusion outputs."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from tests import cobra_generate_reference as gr  # noqa: E402
from tests import cobra_params as cp  # noqa: E402
from tests import cobra_ref  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "cobra_generate.pt")
MARGIN = 5e-2
TRIES = 50
KS = (4, 20)
FULL_ITEMS = (20, 20, 20)
FUSION = dict(n_candidates=10, n_beam=20, temperature=1.0, alpha=0.5)


def calls(cfg, batch_seed):
    """[(name, input_ids, encoder_input_ids)]: each ragged user alone, then the full-length batch"""
    C = cfg["n_codebooks"]
    ids, text = cp.batch(cfg, seed=batch_seed)
    out = [(f"user{b}", ids[b:b + 1, :n * C], text[b:b + 1, :n]) for b, n in enumerate(cp.ITEMS)]
    fids, ftext = cp.batch(cfg, items=FULL_ITEMS, seed=batch_seed + 1)
    return out + [("full", fids, ftext)]


def min_lead(P64, cfg, batch_seed):
    lead = float("inf")
    for _, ids, text in calls(cfg, batch_seed):
        for K in KS:
            g = gr.generate(P64, cfg, ids, text, K)
            lead = min(lead, min(min(x) for x in g["leads"]))
    return lead


def fixture(cfg, first_seed):
    shapes = cp.shapes(cfg)
    for k in range(TRIES):
        seed = first_seed + k
        P = gr.gen_params(cp.cobra_params(shapes, seed))
        lead = min_lead({n: v.double() if v.is_floating_point() else v for n, v in P.items()}, cfg, seed)
        if lead >= MARGIN:
            break
    else:
        raise RuntimeError("no seed with the required margin")
    print("seed", seed, "lead", lead)
    m = cobra_ref.ref_model(cfg, P)
    # LightT5Encoder returns [B, D] for a single item (genrec/modules/encoder.py:103), which generate then reads as D items: the
    # one-item user alone needs its [B, 1, D]
    enc = m.encoder.forward
    m.encoder.forward = lambda tok: enc(tok).view(tok.shape[0], tok.shape[1], -1) if tok.dim() == 3 else enc(tok)
    out = dict(cfg=cfg, param_seed=seed, batch_seed=seed, lead=lead, calls={})
    with torch.no_grad():
        for name, ids, text in calls(cfg, seed):
            for K in KS:
                r = m.generate(ids, text, n_candidates=K)
                out["calls"][f"{name}_k{K}"] = dict(sem_ids=r.sem_ids.clone(), dense_vecs=r.dense_vecs.clone(), scores=r.scores.clone())
        _, fids, ftext = calls(cfg, seed)[-1]
        dense = m.generate(fids, ftext, n_candidates=FUSION["n_beam"]).dense_vecs[:, 0]
        vecs, sem = gr.catalog(cfg, dense, seed)
        r = m.beam_fusion(fids, ftext, vecs, sem, **FUSION)
        P64 = {n: v.double() if v.is_floating_point() else v for n, v in P.items()}
        ref = gr.beam_fusion(P64, cfg, fids, ftext, vecs.double(), sem, **FUSION)
    out["fusion"] = dict(item_ids=r.item_ids.clone(), sem_ids=r.sem_ids.clone(), scores=r.scores.clone(), leads=ref["leads"].float(),
                         sim_leads=ref["sim_leads"].float(), catalog_seed=seed, **FUSION)
    return out


def main(path=OUT):
    assert ref_loader.available(), "reference tree not found"
    torch.save(dict(small=fixture(dict(cp.SMALL), 500), trainer=fixture(dict(cp.TRAINER), 700)), path)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main(*sys.argv[1:])
