"""Generate tests/golden/rqvae_train*.pt from the UNMODIFIED reference (needs the reference tree, see oracle/ref_loader.py).

    TORCHDYNAMO_DISABLE=1 python scripts/make_golden_rqvae_train.py

The reference's ``RqVae.forward`` is wrapped by ``torch.compile``; it runs eagerly here on the CPU.  Eagerly, its ``_sinkhorn_knopp``
multiplies the fp64 kernel matrix with the fp32 ``v = ones`` of its fp32 marginals and raises a dtype error (the compiled graph promotes
that product to fp64).  The recording wrapper below therefore hands the reference's own function its marginals widened to fp64: the same
values, since fp32 -> fp64 is exact, and the product the compiled graph computes.  Every other operation is the reference's.

Fixtures (every file under 1 MB; tests/conftest.py merges <stem>.<key>.pt parts into <stem>.pt):
  rqvae_train_sinkhorn.pt   seeded fp32 ``dist`` at B in {1, 300, 1024} (K = 256): the reference's ids; P at B = 300
  rqvae_train_kmeans.pt     Kmeans(k=64).run on 2,000 seeded rows with seeded numpy / torch RNG: centroids, iterations
  rqvae_train_step.pt       one training forward + backward at TIGER geometry, B = 256, STE / STE / SINKHORN, k-means off
  rqvae_train_step_kmeans.pt  the same model with k-means on, B = 1,024: the post-init codebooks and the outputs
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from tests import rqvae_train_oracle as O  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
TIGER = dict(input_dim=768, hidden=[512, 256, 128, 64], D=32, levels=3, K=256)
BIG = 100_000          # gradients of larger parameters are stored at GRAD_SAMPLES seeded positions
GRAD_SAMPLES = 20_000


def grad_positions(numel: int, seed: int) -> torch.Tensor:
    return torch.randperm(numel, generator=torch.Generator().manual_seed(seed))[:GRAD_SAMPLES].sort().values


def _recorder(rq, log):
    orig = rq._sinkhorn_knopp

    def rec(cost, row_marginals, col_marginals, eps=0.05, max_iter=50):
        P = orig(cost, row_marginals.double(), col_marginals.double(), eps=eps, max_iter=max_iter)
        log.append(P)
        return P

    rq._sinkhorn_knopp = rec


def golden_sinkhorn(rq):
    log = []
    _recorder(rq, log)
    out, parts = {}, {}
    for B, seed in ((1, 200), (300, 201), (1024, 202)):
        torch.manual_seed(seed)
        q = rq.Quantize(embed_dim=32, n_embed=256, do_kmeans_init=False, forward_mode=rq.QuantizeForwardMode.SINKHORN).train()
        g = torch.Generator().manual_seed(seed)
        x = torch.randn(B, 32, generator=g) * 0.3
        with torch.no_grad():
            q.embedding.weight.copy_(torch.randn(256, 32, generator=g) * 0.3)
            q.embedding.weight[77] = q.embedding.weight[5]          # identical codes: the lower index must win
            dist = (x ** 2).sum(axis=1, keepdim=True) + (q.embedding.weight.T ** 2).sum(axis=0, keepdim=True) - 2 * x @ q.embedding.weight.T
            log.clear()
            ids = q(x, temperature=0.2).ids
        assert torch.equal(ids, log[0].argmax(-1))
        out[f"ids{B}"] = ids.clone()
        if B == 1024:
            parts["dist1024a"], parts["dist1024b"] = dist[:512].clone(), dist[512:].clone()
        else:
            out[f"dist{B}"] = dist.clone()
        if B == 300:
            parts["P300"] = log[0].clone()
    torch.save(out, os.path.join(OUT, "rqvae_train_sinkhorn.pt"))
    for k, v in parts.items():
        torch.save(v, os.path.join(OUT, f"rqvae_train_sinkhorn.{k}.pt"))


def golden_kmeans():
    km = ref_loader._ref_module("genrec.modules.kmeans")
    g = torch.Generator().manual_seed(300)
    centres = torch.randn(64, 32, generator=g)
    x = centres[torch.randint(0, 64, (2000,), generator=g)] + 0.2 * torch.randn(2000, 32, generator=g)
    np.random.seed(301)
    torch.manual_seed(302)
    k = km.Kmeans(k=64)
    c = k.run(x).centroids
    # the converging iteration, counted the way kmeans.py:88-94 counts, from a second identically seeded run
    np.random.seed(301)
    torch.manual_seed(302)
    _, it, init = O.kmeans(x, 64)
    np.random.seed(301)
    init_ref = np.random.choice(2000, 64, replace=False)
    torch.save(dict(x=x, np_seed=301, torch_seed=302, k=64, centroids=c.clone(), init_rows=torch.from_numpy(init_ref)),
               os.path.join(OUT, "rqvae_train_kmeans.pt"))
    print("kmeans: oracle iterations", it, "same init", bool((init == init_ref).all()))


def _ref_model(rq, kmeans):
    return rq.RqVae(input_dim=TIGER["input_dim"], embed_dim=TIGER["D"], hidden_dims=TIGER["hidden"], codebook_size=TIGER["K"],
                    codebook_kmeans_init=kmeans, codebook_mode=rq.QuantizeForwardMode.STE,
                    codebook_last_layer_mode=rq.QuantizeForwardMode.SINKHORN, n_layers=TIGER["levels"], n_cat_features=0)


def golden_step(rq):
    log = []
    _recorder(rq, log)
    state = O.seeded_state(TIGER["input_dim"], TIGER["hidden"], TIGER["D"], TIGER["levels"], TIGER["K"], seed=400)
    x = O.seeded_items(256, TIGER["input_dim"], seed=401)
    m = _ref_model(rq, False).train()
    m.load_state_dict(state, strict=True)
    out = m(x, 0.2)
    out.loss.backward()
    ids = [None] * 3
    with torch.no_grad():                      # the ids each level used: STE levels from their argmin, the last from P
        sem = m.get_semantic_ids(x).sem_ids
        ids[0], ids[1] = sem[:, 0].clone(), sem[:, 1].clone()
    ids[2] = log[0].argmax(-1)
    grads = {}
    for n, p in m.named_parameters():
        gr = p.grad.detach().flatten()
        grads[n] = gr[grad_positions(gr.numel(), 402)].clone() if gr.numel() > BIG else p.grad.detach().clone()
    torch.save(dict(state_seed=400, items_seed=401, grad_seed=402, B=256,
                    outputs={k: v.detach().clone() for k, v in out._asdict().items()}, ids=ids),
               os.path.join(OUT, "rqvae_train_step.pt"))
    torch.save(grads, os.path.join(OUT, "rqvae_train_step.grads.pt"))


def golden_step_kmeans(rq):
    _recorder(rq, [])
    state = O.seeded_state(TIGER["input_dim"], TIGER["hidden"], TIGER["D"], TIGER["levels"], TIGER["K"], seed=400)
    x = O.seeded_items(1024, TIGER["input_dim"], seed=403)
    m = _ref_model(rq, True).train()
    m.load_state_dict(state, strict=True)
    np.random.seed(404)
    torch.manual_seed(405)
    out = m(x, 0.2)
    torch.save(dict(state_seed=400, items_seed=403, np_seed=404, torch_seed=405, B=1024,
                    codebooks=torch.stack([l.embedding.weight.detach().clone() for l in m.layers]),
                    outputs={k: v.detach().clone() for k, v in out._asdict().items()}),
               os.path.join(OUT, "rqvae_train_step_kmeans.pt"))


def main():
    assert ref_loader.available(), "reference tree not found"
    assert os.environ.get("TORCHDYNAMO_DISABLE") == "1", "run with TORCHDYNAMO_DISABLE=1 (the reference's forward is torch.compile'd)"
    rq = ref_loader.ref_genrec_package().rqvae
    golden_sinkhorn(rq)
    golden_kmeans()
    golden_step(rq)
    golden_step_kmeans(rq)
    for f in sorted(os.listdir(OUT)):
        if f.startswith("rqvae_train"):
            print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()
