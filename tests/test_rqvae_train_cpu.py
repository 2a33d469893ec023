"""RQ-VAE training path without a GPU: the restatement (tests/rqvae_train_oracle.py) against the reference's fixtures, the C ABI's
refusals, and the tolerances of test_rqvae_train_gpu.py against restatements of Sinkhorn with deliberate mistakes."""
import ctypes

import numpy as np
import pytest
import torch

from tests import rqvae_train_oracle as O

TIGER = dict(input_dim=768, hidden=[512, 256, 128, 64], D=32, levels=3, K=256)
MODES = ["STE", "STE", "SINKHORN"]
UV_TOL = 1e-9          # test_rqvae_train_gpu.py: u and v, relative per entry
MARGIN = 3.0


def _dist(g, B):
    return g["rqvae_train_sinkhorn.pt"][f"dist{B}"] if B != 1024 else torch.cat([g["rqvae_train_sinkhorn.pt"]["dist1024a"],
                                                                                   g["rqvae_train_sinkhorn.pt"]["dist1024b"]])


@pytest.fixture(scope="module")
def fx(golden):
    return {n: golden(n) for n in ("rqvae_train_sinkhorn.pt", "rqvae_train_kmeans.pt", "rqvae_train_step.pt", "rqvae_train_step_kmeans.pt")}


@pytest.mark.parametrize("B", [1, 300, 1024])
def test_oracle_sinkhorn_matches_reference(fx, B):
    ids, u, v, P = O.sinkhorn(_dist(fx, B))
    assert torch.equal(ids, fx["rqvae_train_sinkhorn.pt"][f"ids{B}"])
    if B == 300:
        ref = fx["rqvae_train_sinkhorn.pt"]["P300"]
        assert ((P - ref).abs() <= 1e-15 * ref.abs()).all()


def test_oracle_kmeans_matches_reference(fx):
    k = fx["rqvae_train_kmeans.pt"]
    np.random.seed(k["np_seed"])
    torch.manual_seed(k["torch_seed"])
    c, it, init = O.kmeans(k["x"], k["k"])
    assert np.array_equal(init, k["init_rows"].numpy())
    assert (c - k["centroids"]).abs().max() <= 1e-6


def _step_inputs(s, B):
    p = O.seeded_state(TIGER["input_dim"], TIGER["hidden"], TIGER["D"], TIGER["levels"], TIGER["K"], seed=s["state_seed"])
    return p, O.seeded_items(B, TIGER["input_dim"], seed=s["items_seed"])


def _close(a, b, tol=1e-6):
    a = a.detach()
    return float((a - b).abs().max()) <= tol * max(1.0, float(b.abs().max()))


def test_oracle_training_step_matches_reference(fx):
    from scripts.make_golden_rqvae_train import BIG, grad_positions
    s = fx["rqvae_train_step.pt"]
    p, x = _step_inputs(s, s["B"])
    p = {k: v.clone().requires_grad_(True) for k, v in p.items()}
    out, ids = O.train_forward(p, x, MODES)
    for lv in range(3):
        assert torch.equal(ids[lv], s["ids"][lv]), lv
    for k, ref in s["outputs"].items():
        assert _close(out[k].float(), ref.float()), k
    out["loss"].backward()
    for n, ref in s["grads"].items():
        gr = p[n].grad.flatten()
        if gr.numel() > BIG:
            gr = gr[grad_positions(gr.numel(), s["grad_seed"])]
        assert float((gr - ref.flatten()).abs().max()) <= 1e-6 * float(ref.abs().max()), n


def oracle_kmeans_levels(p, x, np_seed, torch_seed, modes=MODES):
    """The first RqVae.forward with k-means on: every level initialises its codebook on its input residual, then quantises."""
    np.random.seed(np_seed)
    torch.manual_seed(torch_seed)
    res = O.mlp(x, O._weights(p, "encoder"), False)
    cbs = []
    for lv, mode in enumerate(modes):
        cb = O.kmeans(res, p[f"layers.{lv}.embedding.weight"].shape[0])[0]
        cbs.append(cb)
        dist = O.l2_dist(res, cb)
        ids = O.sinkhorn(dist)[0] if mode == "SINKHORN" else dist.min(1).indices
        res = res - cb[ids]
    return torch.stack(cbs)


def test_oracle_kmeans_init_matches_reference(fx):
    s = fx["rqvae_train_step_kmeans.pt"]
    p, x = _step_inputs(s, s["B"])
    with torch.no_grad():
        cbs = oracle_kmeans_levels(p, x, s["np_seed"], s["torch_seed"])
    assert (cbs - s["codebooks"]).abs().max() <= 1e-6


def test_p_unique_ids_matches_the_pairwise_definition():
    from genrec_b200.rqvae import p_unique_ids
    g = torch.Generator().manual_seed(0)
    for B, levels, K in ((1, 3, 256), (500, 3, 4), (300, 5, 256), (64, 2, 2)):
        sem = torch.randint(0, K, (B, levels), generator=g)
        sem[B // 2:] = sem[: B - B // 2]                  # duplicates
        same = (sem[:, None, :] == sem[None, :, :]).all(-1)
        ref = (~torch.triu(same, diagonal=1)).all(1).sum() / B
        got = p_unique_ids(sem, K)
        assert got.dtype == ref.dtype and torch.equal(got, ref)
    with pytest.raises(NotImplementedError):
        p_unique_ids(torch.zeros(4, 8, dtype=torch.int64), 256)


# ---------------------------------------------------------------------------------------------------- C ABI refusals, no GPU
@pytest.fixture(scope="module")
def lib():
    from genrec_b200 import build
    build.build()
    from genrec_b200 import _lib
    return _lib.load()


def test_sinkhorn_workspace_query(lib):
    # B = 1024, K = 256: a CTA's 64 rows of K fit shared memory, the workspace holds u only; B = 20,480 adds the fp64 [B, K] matrix
    assert lib.grb_rq_sinkhorn_workspace_bytes(1024, 256) == 1024 * 8
    assert lib.grb_rq_sinkhorn_workspace_bytes(20480, 256) == 20480 * 8 + 20480 * 256 * 8
    assert lib.grb_rq_sinkhorn_workspace_bytes(0, 32) == 0
    for B, K in ((10, 1), (10, 257), (-1, 32)):
        assert lib.grb_rq_sinkhorn_workspace_bytes(B, K) == 0
        assert b"unsupported" in lib.grb_last_error()


def test_sinkhorn_refusals(lib):
    buf = (ctypes.c_char * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p).value
    for B, K, eps, iters in ((8, 1, 0.003, 100), (8, 257, 0.003, 100), (-1, 32, 0.003, 100), (8, 32, 0.0, 100), (8, 32, 0.003, -1)):
        assert lib.grb_rq_sinkhorn(p, B, K, eps, iters, p, None, None, p, None) == -1, (B, K, eps, iters)
        assert b"unsupported" in lib.grb_last_error()
    assert lib.grb_rq_sinkhorn(None, 8, 32, 0.003, 100, p, None, None, p, None) == -1
    assert b"null" in lib.grb_last_error()
    assert lib.grb_rq_sinkhorn(p, 8, 32, 0.003, 100, None, None, None, p, None) == -1
    assert lib.grb_rq_sinkhorn(p, 8, 32, 0.003, 100, p, None, None, None, None) == -1
    assert lib.grb_rq_sinkhorn(None, 0, 32, 0.003, 100, None, None, None, None, None) == 0       # B = 0: nothing to do


def test_kmeans_update_refusals(lib):
    buf = (ctypes.c_char * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p).value
    for B, D, k in ((-1, 32, 8), (10, 0, 8), (10, 257, 8), (10, 32, 0)):
        assert lib.grb_kmeans_update(p, p, B, D, k, p, p, p, None) == -1, (B, D, k)
        assert b"unsupported" in lib.grb_last_error()
    for i in range(5):
        args = [p, p, 10, 32, 8, p, p, p, None]
        args[[0, 1, 5, 6, 7][i]] = None
        assert lib.grb_kmeans_update(*args) == -1
        assert b"null" in lib.grb_last_error()


# ---------------------------------------------------------------------------------------------------- mutations
MUTATIONS = {
    "iters99": dict(iters=99),
    "eps0.03": dict(eps=0.03),
    "fp64_marginals": dict(fp32_marginals=False),
    "swapped_updates": dict(swap=True),
    "rowwise_normalisation": dict(rowwise=True),
    "no_1e-8": dict(stab=0.0),
}


def _uv_excess(mut, ref):
    """How many GPU tolerances (relative, per entry) the mutated u, v land from the correct ones."""
    return max(float(((m - r).abs() / r.abs()).max()) for m, r in zip(mut[1:3], ref[1:3])) / UV_TOL


def _mutation_inputs(fx):
    g = torch.Generator().manual_seed(7)
    x, cb = torch.randn(255, 32, generator=g), torch.randn(32, 32, generator=g)
    return {"B300": _dist(fx, 300), "B1024": _dist(fx, 1024), "B255K32": O.l2_dist(x, cb)}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
@pytest.mark.parametrize("case", ["B300", "B1024", "B255K32"])
def test_tolerances_catch_sinkhorn_mistakes(fx, case, mutation):
    dist = _mutation_inputs(fx)[case]
    B, K = dist.shape
    if mutation == "fp64_marginals" and all(float(np.float32(1.0 / n)) == 1.0 / n for n in (B, K)):
        pytest.skip("1/B and 1/K are exact in fp32: the rounding changes nothing")
    ref = O.sinkhorn(dist)
    mut = O.sinkhorn(dist, **{"eps": O.EPS, "iters": O.ITERS, **MUTATIONS[mutation]})
    assert _uv_excess(mut, ref) >= MARGIN
