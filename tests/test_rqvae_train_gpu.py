"""RQ-VAE training on the GPU: rq_sinkhorn against the fp64 restatement, the device k-means against the restated reference loop,
RqVae.forward against the restatement and the reference's fixtures, and a short training run (tests/rqvae_train_oracle.py)."""
import numpy as np
import pytest
import torch

from tests import rqvae_train_oracle as O

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
UV_TOL = 1e-9
GAP_TOL = 1e-9
GEOMS = {"tiger": dict(input_dim=768, hidden=[512, 256, 128, 64], D=32, levels=3, K=256),
         "lcrec": dict(input_dim=768, hidden=[512, 256, 128], D=64, levels=5, K=256)}


def _dist(B, K, seed):
    g = torch.Generator().manual_seed(seed)
    x, cb = torch.randn(B, 32, generator=g) * 0.3, torch.randn(K, 32, generator=g) * 0.3
    return O.l2_dist(x, cb)


def _check_sinkhorn(dist, label=""):
    import genrec_b200.functional as Fn
    ids, u, v = Fn.rq_sinkhorn(dist.to(DEV))
    rid, ru, rv, P = O.sinkhorn(dist)
    for got, ref in ((u.cpu(), ru), (v.cpu(), rv)):
        rel = float(((got - ref).abs() / ref.abs()).max())
        assert rel <= UV_TOL, (label, rel)
    top2 = P.topk(2, dim=1).values if P.shape[1] > 1 else None
    decided = (top2[:, 0] - top2[:, 1]) > GAP_TOL * top2[:, 0]
    print(f"{label}: {int((~decided).sum())} of {len(decided)} rows within a {GAP_TOL:g} relative top-2 gap")
    assert torch.equal(ids.cpu()[decided], rid[decided]), label
    return ids


@pytest.mark.parametrize("K", [32, 256])
@pytest.mark.parametrize("B", [1, 2, 7, 255, 1000, 1024, 20480])
def test_sinkhorn_matches_oracle(B, K):
    _check_sinkhorn(_dist(B, K, seed=B * 3 + K), f"B={B} K={K}")


def test_sinkhorn_on_reference_fixtures(golden):
    g = golden("rqvae_train_sinkhorn.pt")
    for B in (1, 300, 1024):
        dist = g[f"dist{B}"] if B != 1024 else torch.cat([g["dist1024a"], g["dist1024b"]])
        ids = _check_sinkhorn(dist, f"fixture B={B}")
        assert (ids.cpu() == g[f"ids{B}"]).float().mean() >= 0.999


def test_sinkhorn_edge_cases():
    import genrec_b200.functional as Fn
    # two identical codes (identical distance columns), with rows near them: the lower index wins
    g = torch.Generator().manual_seed(1)
    x, cb = torch.randn(600, 32, generator=g), torch.randn(256, 32, generator=g)
    x[:60] = cb[17] + 0.01 * torch.randn(60, 32, generator=g)
    dist = O.l2_dist(x, cb)
    dist[:, 200] = dist[:, 17]
    ids = _check_sinkhorn(dist, "duplicate code")
    assert not (ids == 200).any() and (ids == 17).any()
    # all distances equal: amp = 1e-5, every K_ij = 1, ids all 0
    ids, u, v = Fn.rq_sinkhorn(torch.full((300, 64), 2.5, device=DEV))
    assert (ids == 0).all() and torch.isfinite(u).all() and torch.isfinite(v).all()
    # B = 0
    assert Fn.rq_sinkhorn(torch.empty(0, 32, device=DEV))[0].shape == (0,)
    with pytest.raises(RuntimeError):
        Fn.rq_sinkhorn(torch.zeros(4, 257, device=DEV))


@pytest.mark.parametrize("B", [1024, 20480])
def test_sinkhorn_is_deterministic_and_graph_capturable(B):
    import genrec_b200.functional as Fn
    d1, d2 = _dist(B, 256, 11).to(DEV), _dist(B, 256, 12).to(DEV)
    a = Fn.rq_sinkhorn(d1)
    b = Fn.rq_sinkhorn(d1)
    assert all(torch.equal(p, q) for p, q in zip(a, b))
    buf = d1.clone()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        Fn.rq_sinkhorn(buf)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            out = Fn.rq_sinkhorn(buf)
    buf.copy_(d2)
    graph.replay()
    torch.cuda.synchronize()
    eager = Fn.rq_sinkhorn(d2)
    assert all(torch.equal(p, q) for p, q in zip(out, eager))


def test_sinkhorn_custom_op():
    import genrec_b200.ops  # noqa: F401
    import genrec_b200.functional as Fn
    d = _dist(100, 64, 3).to(DEV)
    assert all(torch.equal(p, q) for p, q in zip(torch.ops.genrec_b200.rq_sinkhorn(d, 0.003, 100), Fn.rq_sinkhorn(d)))


# ---------------------------------------------------------------------------------------------------- k-means
def _mixture(B, k, D, seed, spread=0.1):
    """k blobs of B / k rows around N(0, 1) centres: blobs about 8 apart, rows about 0.6 from their centre.  The search computes
    |x|^2 + |c|^2 - 2 x.c where the reference sums (x - c)^2; at |x|^2 ~ 32 the two differ by ~1e-5, far below any distance
    between a row and two centroids in different blobs."""
    g = torch.Generator().manual_seed(seed)
    centres = torch.randn(k, D, generator=g)
    return centres[torch.arange(B) % k] + spread * torch.randn(B, D, generator=g)


def _run_both(x, k, np_seed, torch_seed, oracle_device):
    from genrec_b200.rqvae import kmeans_init_
    w = torch.empty(k, x.shape[1], device=DEV)
    np.random.seed(np_seed)
    torch.manual_seed(torch_seed)
    it = kmeans_init_(w, x.to(DEV))
    ours_next = (np.random.rand(), torch.rand(1))
    np.random.seed(np_seed)
    torch.manual_seed(torch_seed)
    c, it_ref, _ = O.kmeans(x.to(oracle_device), k)
    ref_next = (np.random.rand(), torch.rand(1))
    assert ours_next[0] == ref_next[0] and torch.equal(ours_next[1], ref_next[1]), "RNG consumption differs"
    return w.cpu(), it, c.cpu(), it_ref


def test_kmeans_matches_reference_loop_on_a_mixture():
    x = _mixture(20480, 256, 32, seed=5)
    w, it, c, it_ref = _run_both(x, 256, 6, 7, DEV)
    print(f"k-means: {it} iterations (restated reference {it_ref})")
    assert it == it_ref
    assert (w - c).abs().max() <= 1e-5


def test_kmeans_reseeds_empty_clusters_like_the_reference():
    g = torch.Generator().manual_seed(8)
    base = torch.randint(-8, 8, (80, 32), generator=g) / 4.0     # dyadic values: every cluster mean is exact in fp32 and fp64
    x = base[torch.randint(0, 80, (2000,), generator=g)]          # 80 distinct rows, duplicated: initial draws collide
    w, it, c, it_ref = _run_both(x, 64, 9, 10, "cpu")
    assert it == it_ref
    assert (w - c).abs().max() <= 1e-5


def test_kmeans_refusals():
    from genrec_b200.rqvae import KMEANS_MAX_ITERS, kmeans_init_
    assert KMEANS_MAX_ITERS == 10_000
    w = torch.empty(64, 32, device=DEV)
    with pytest.raises(ValueError):
        kmeans_init_(w, torch.randn(63, 32, device=DEV))
    x = torch.randn(10, 32, device=DEV)[torch.arange(300, device=DEV) % 10]   # 10 distinct rows < k: never converges
    with pytest.raises(RuntimeError, match="did not converge"):
        kmeans_init_(w, x)


# ---------------------------------------------------------------------------------------------------- RqVae.forward
def _model(geo, kmeans=False, seed=400):
    from genrec_b200.rqvae import QuantizeForwardMode as M, RqVae
    m = RqVae(input_dim=geo["input_dim"], embed_dim=geo["D"], hidden_dims=geo["hidden"], codebook_size=geo["K"], codebook_kmeans_init=kmeans,
              codebook_mode=M.STE, codebook_last_layer_mode=M.SINKHORN, n_layers=geo["levels"], n_cat_features=0)
    state = O.seeded_state(geo["input_dim"], geo["hidden"], geo["D"], geo["levels"], geo["K"], seed)
    m.load_state_dict(state, strict=True)
    return m.to(DEV), state


def _rel(a, b):
    return float((a.detach().cpu().double() - b.detach().double()).abs().max() / max(b.detach().double().abs().max(), 1e-30))


@pytest.mark.parametrize("geo", ["tiger", "lcrec"])
def test_training_forward_matches_oracle(geo):
    G = GEOMS[geo]
    modes = ["STE"] * (G["levels"] - 1) + ["SINKHORN"]
    m, state = _model(G)
    x = O.seeded_items(1024, G["input_dim"], seed=41)
    m.train()
    out = m(x.to(DEV), 0.2)
    out.loss.backward()
    ref, ref_ids = O.train_forward(state, x, modes)
    for k in ("loss", "reconstruction_loss", "rqvae_loss"):
        assert _rel(getattr(out, k), ref[k]) <= 1e-4, k
    # the forward's ids level by level, recomputed with the same operations on the same values (STE: emb_out = x + (emb - x))
    import genrec_b200.functional as Fn
    res = m.encode(x.to(DEV)).detach()
    ids = []
    for lv, layer in enumerate(m.layers):
        cb = layer.embedding.weight.detach()
        idl = Fn.rq_sinkhorn(O.l2_dist(res, cb))[0] if modes[lv] == "SINKHORN" else \
            Fn.rq_residual_argmin(res, cb.unsqueeze(0), want_aux=False)[0][:, 0]
        ids.append(idl.cpu())
        res = res - (res + (cb[idl] - res))
    agree = float((torch.stack(ids, -1) == torch.stack(ref_ids, -1)).all(-1).float().mean())
    print(f"{geo}: sem_ids agree on {agree:.4f} of rows")
    assert agree >= 0.99
    # gradients, embs_norm and p_unique_ids given the GPU's ids
    p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    ref2, _ = O.train_forward(p, x, modes, ids=ids)
    ref2["loss"].backward()
    for n, par in m.named_parameters():
        assert _rel(par.grad, p[n].grad) <= 1e-4, n
    assert _rel(out.embs_norm, ref2["embs_norm"]) <= 1e-6
    assert float(out.p_unique_ids) == float(ref2["p_unique_ids"])
    # eval mode
    m.eval()
    with torch.no_grad():
        ev = m(x.to(DEV), 0.2)
    ref_ev, _ = O.train_forward(state, x, modes, training=False)
    for k in ("loss", "reconstruction_loss", "rqvae_loss"):
        assert _rel(getattr(ev, k), ref_ev[k]) <= 1e-4, k
    assert abs(float(ev.p_unique_ids) - float(ref_ev["p_unique_ids"])) <= 0.01


def test_training_step_matches_reference_fixture(golden):
    s = golden("rqvae_train_step.pt")
    m, _ = _model(GEOMS["tiger"], seed=s["state_seed"])
    x = O.seeded_items(s["B"], 768, seed=s["items_seed"]).to(DEV)
    out = m.train()(x, 0.2)
    for k, ref in s["outputs"].items():
        if k == "embs_norm":
            continue
        assert _rel(getattr(out, k), ref) <= 1e-4, k
    with torch.no_grad():
        sem = m.get_semantic_ids(x).sem_ids.cpu()
    assert float((sem[:, :2] == torch.stack(s["ids"][:2], -1)).all(-1).float().mean()) >= 0.99


def test_kmeans_init_matches_reference_fixture(golden):
    s = golden("rqvae_train_step_kmeans.pt")
    m, _ = _model(GEOMS["tiger"], kmeans=True, seed=s["state_seed"])
    x = O.seeded_items(s["B"], 768, seed=s["items_seed"]).to(DEV)
    np.random.seed(s["np_seed"])
    torch.manual_seed(s["torch_seed"])
    m.train()(x, 0.2)
    assert all(l.kmeans_initted for l in m.layers)
    cbs = m.codebooks().detach().cpu()
    close = ((cbs - s["codebooks"]).abs().amax(-1) <= 1e-4).float().mean(-1)
    print("k-means fixture: fraction of codebook rows within 1e-4 per level", close.tolist())
    assert close[0] >= 0.99 and close.min() >= 0.9


def test_forward_has_no_host_sync_after_kmeans():
    m, _ = _model(GEOMS["tiger"], kmeans=True)
    x = O.seeded_items(1024, 768, seed=42).to(DEV)
    m.train()(x, 0.2)                               # k-means (host reads) happens here
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = m(x, 0.2)
        out.loss.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)


# ---------------------------------------------------------------------------------------------------- short training run
def _train(model_fn, params, items, steps=300, B=1024, seed=0):
    """rqvae_trainer.py:160-240: AdamW(lr 1e-3, wd 1e-4), linear warm-up, clip_grad_norm_(1.0), k-means on the first batch."""
    opt = torch.optim.AdamW(params, lr=1e-3, weight_decay=1e-4)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda s: min(1.0, (s + 1) / 30) * max(0.0, (steps - s) / steps))
    g = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        batch = items[torch.randint(0, len(items), (B,), generator=g).to(items.device)]
        opt.zero_grad()
        rec = model_fn(batch)
        torch.nn.utils.clip_grad_norm_(params, 1.0)
        opt.step()
        sched.step()
    return float(rec)


def _collision(sem):
    return 1.0 - len({tuple(r) for r in sem.tolist()}) / len(sem)


def test_short_training_run_against_torch_restatement():
    G = GEOMS["tiger"]
    modes = ["STE", "STE", "SINKHORN"]
    items = O.seeded_items(20480, 768, seed=50, n_clusters=512).to(DEV)
    results = {}
    # ours
    m, state = _model(G, kmeans=False, seed=51)
    m.train()

    def ours(batch):
        out = m(batch, 0.2)
        out.loss.backward()
        return out.reconstruction_loss.detach()

    rec = _train(ours, list(m.parameters()), items)
    with torch.no_grad():
        m.eval()
        final = m(items, 0.2).reconstruction_loss
        sem = m.get_semantic_ids(items).sem_ids
    results["ours"] = (float(final), _collision(sem.cpu()))
    # the torch restatement in fp32 and in fp64, same initial state and batches
    for dt in (torch.float32, torch.float64):
        p = {k: v.to(DEV, dt).requires_grad_(True) for k, v in state.items()}

        def ref(batch):
            out, _ = O.train_forward(p, batch.to(dt), modes)
            out["loss"].backward()
            return out["reconstruction_loss"].detach()

        _train(ref, list(p.values()), items)
        with torch.no_grad():
            out, ids = O.train_forward(p, items.to(dt), modes, training=False)
        results[str(dt)] = (float(out["reconstruction_loss"]), _collision(torch.stack(ids, -1).cpu()))
    print("short run (final reconstruction loss, collision rate):", results)
    (r32, c32), (r64, c64), (ro, co) = results["torch.float32"], results["torch.float64"], results["ours"]
    assert abs(ro - r32) <= 3 * max(abs(r32 - r64), 1e-3 * abs(r64)), results
    assert abs(co - c32) <= 3 * max(abs(c32 - c64), 0.01), results
