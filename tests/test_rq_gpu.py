import pytest
import torch

pytestmark = pytest.mark.gpu


def test_rq_vs_reference_golden(golden):
    from genrec_b200.rqvae import RqVae
    g = golden("rqvae_3x256x32.pt")
    cfg = g["cfg"]
    dev = torch.device("cuda:0")
    m = RqVae(cfg["input_dim"], cfg["D"], cfg["hidden_dims"], cfg["K"], codebook_kmeans_init=False, n_layers=cfg["levels"],
              n_cat_features=0)
    missing = m.load_state_dict(g["state_dict"], strict=False)
    assert all(k.startswith("decoder") for k in missing.missing_keys) and not missing.unexpected_keys
    m = m.to(dev).eval()
    # 1) from the reference latent: ids bit-exact, incl. the duplicated-code ties
    import genrec_b200.functional as Fn
    ids, emb, res, loss = Fn.rq_residual_argmin(g["latent"].to(dev), m.codebooks(), 0.25)
    assert torch.equal(ids.cpu(), g["sem_ids"])
    assert torch.equal(emb.cpu(), g["embeddings"])
    torch.testing.assert_close(res.cpu(), g["residuals"], rtol=0, atol=1e-6)
    torch.testing.assert_close(loss.cpu(), g["quantize_loss"], rtol=1e-5, atol=1e-6)
    # 2) end to end (encoder on cuBLAS may flip a near-tie): ids agree on >= 99% of rows
    out = m.get_semantic_ids(g["x"].to(dev))
    assert out.sem_ids.shape == g["sem_ids"].shape and out.embeddings.shape == g["embeddings"].shape
    agree = (out.sem_ids.cpu() == g["sem_ids"]).all(1).float().mean().item()
    assert agree >= 0.99, agree


@pytest.mark.parametrize("N,D,K,levels", [(12101, 32, 256, 3), (1, 32, 256, 3), (257, 64, 256, 5), (1 << 20, 32, 256, 3)])
def test_rq_vs_oracle_and_properties(N, D, K, levels):
    import genrec_b200.functional as Fn
    from oracle import rqvae as orq
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(N % 1000 + D)
    x = torch.randn(N, D, generator=g)
    cbs = torch.stack([(torch.rand(K, D, generator=g) - 0.5) * (2.0 / 2 ** l) for l in range(levels)])
    ids, emb, res, loss = Fn.rq_residual_argmin(x.to(dev), cbs.to(dev), 0.25)
    ids, emb, res, loss = ids.cpu(), emb.cpu(), res.cpu(), loss.cpu()
    # properties at any size: residual recursion and optimality of every chosen code
    r = x.clone()
    for l in range(levels):
        torch.testing.assert_close(res[:, :, l], r, rtol=0, atol=1e-5)
        e = cbs[l][ids[:, l]]
        assert torch.equal(emb[:, :, l], e)
        if N <= 20000:
            d = torch.cdist(r.double(), cbs[l].double()) ** 2
            chosen = d.gather(1, ids[:, l:l + 1]).squeeze(1)
            assert (chosen <= d.min(1).values + 1e-4).all()
        r = r - e
    if N <= 20000:
        o = orq.residual_quantize(x, list(cbs))
        agree = (o.sem_ids == ids).all(1).float().mean().item()
        assert agree >= 0.995, agree
        torch.testing.assert_close(loss, o.quantize_loss, rtol=1e-4, atol=1e-5)


def test_rq_empty_and_errors():
    import genrec_b200.functional as Fn
    dev = torch.device("cuda:0")
    ids, *_ = Fn.rq_residual_argmin(torch.zeros(0, 32, device=dev), torch.rand(3, 256, 32, device=dev))
    assert ids.shape == (0, 3)
    with pytest.raises(RuntimeError):
        Fn.rq_residual_argmin(torch.zeros(4, 48, device=dev), torch.rand(3, 256, 48, device=dev))
    with pytest.raises(RuntimeError):
        Fn.rq_residual_argmin(torch.zeros(4, 32), torch.rand(3, 256, 32))


@pytest.mark.parametrize("N,D,levels", [(12101, 32, 3), (777, 64, 5), (200_000, 32, 3), (129, 32, 1), (1, 32, 4)])
def test_rq_kernel_generations_are_bit_identical(N, D, levels, monkeypatch):
    """The register-blocked tile kernel (default where it applies: D = 32, K % 256 == 0), the four-threads-per-row kernel and the
    first-generation one-thread-per-row kernel keep the same arithmetic (same dot-product order, same tie rule): every output is
    bit-identical, including the staged [N, D, levels] writes and ragged last tiles."""
    import genrec_b200.functional as Fn
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(N % 997 + D)
    x = torch.randn(N, D, generator=g).to(dev)
    cbs = torch.stack([(torch.rand(256, D, generator=g) - 0.5) * (2.0 / 2 ** l) for l in range(levels)])
    cbs[0, 200] = cbs[0, 17]                       # exact ties: the first index must win in both
    cbs = cbs.to(dev)
    out = {}
    for mode in ("tile", "split", "thread"):
        monkeypatch.setenv("GRB_RQ", mode)
        out[mode] = Fn.rq_residual_argmin(x, cbs, 0.25)
    for mode in ("tile", "split"):
        for a, b in zip(out[mode], out["thread"]):
            assert torch.equal(a, b), mode
    monkeypatch.delenv("GRB_RQ")
    ids_only = Fn.rq_residual_argmin(x, cbs, 0.25, want_aux=False)[0]
    assert torch.equal(ids_only, out["thread"][0])


def test_rq_encoder_fp32_accurate_tensor_path(golden):
    """RqVae.encode at inference = five wgmma GEMMs on three-term bf16 splits (SiLU in the epilogue): fp32 accuracy against the
    oracle's fp32 MLP, and the semantic ids of the reference golden end to end."""
    from genrec_b200.rqvae import RqVae
    from oracle import rqvae as orq
    g = golden("rqvae_3x256x32.pt")
    cfg = g["cfg"]
    dev = torch.device("cuda:0")
    m = RqVae(cfg["input_dim"], cfg["D"], cfg["hidden_dims"], cfg["K"], codebook_kmeans_init=False, n_layers=cfg["levels"], n_cat_features=0)
    m.load_state_dict(g["state_dict"], strict=False)
    m = m.to(dev).eval()
    with torch.no_grad():
        lat = m.encode(g["x"].to(dev)).cpu()
    torch.testing.assert_close(lat, g["latent"], rtol=2e-5, atol=2e-6)
    out = m.get_semantic_ids(g["x"].to(dev))
    agree = (out.sem_ids.cpu() == g["sem_ids"]).all(1).float().mean().item()
    assert agree >= 0.995, agree
    # the production geometry: 768 -> 512 -> 256 -> 128 -> 64 -> 32 on 12,101 items
    torch.manual_seed(0)
    big = RqVae(768, 32, [512, 256, 128, 64], 256, codebook_kmeans_init=False, n_layers=3, n_cat_features=0).to(dev).eval()
    x = torch.randn(12101, 768)
    x = x / x.norm(dim=1, keepdim=True)
    ws = [l.weight.detach().cpu() for l in big.encoder.mlp if isinstance(l, torch.nn.Linear)]
    ref = orq.mlp_encoder(x.double(), [w.double() for w in ws]).float()
    with torch.no_grad():
        got = big.encode(x.to(dev)).cpu()
    err = ((got - ref).abs().max() / ref.abs().max()).item()
    assert err < 1e-5, err


@pytest.mark.parametrize("mode", ["STE", "ROTATION_TRICK", "GUMBEL_SOFTMAX"])
def test_quantize_training_mode_matches_reference_formulas(mode):
    """Training-mode Quantize.forward (rqvae.py:201-245): ids from the CUDA search, estimator = the reference's formulas."""
    from genrec_b200.rqvae import Quantize, QuantizeForwardMode
    dev = torch.device("cuda:0")
    torch.manual_seed(3)
    q = Quantize(32, 256, do_kmeans_init=False, forward_mode=QuantizeForwardMode[mode]).to(dev).train()
    x = torch.randn(500, 32, device=dev, requires_grad=True)
    out = q(x, 0.2)
    assert out.embeddings.shape == (500, 32) and out.ids.shape == (500,) and out.loss.shape == (500,)
    # ids: nearest code (fp64 check of optimality)
    d = torch.cdist(x.detach().double(), q.embedding.weight.detach().double()) ** 2
    assert (d.gather(1, out.ids[:, None]).squeeze(1) <= d.min(1).values + 1e-5).all()
    (out.embeddings.sum() + out.loss.sum()).backward()
    assert torch.isfinite(x.grad).all() and q.embedding.weight.grad is not None
    if mode == "GUMBEL_SOFTMAX":
        return
    # reference formulas on the CPU with the same ids
    xc = x.detach().cpu().requires_grad_(True)
    cb = q.embedding.weight.detach().cpu().requires_grad_(True)
    emb = cb[out.ids.cpu()]
    if mode == "STE":
        emb_out = xc + (emb - xc).detach()
    else:
        u = xc / (xc.norm(dim=-1, keepdim=True) + 1e-8)
        qq = emb / (emb.norm(dim=-1, keepdim=True) + 1e-8)
        w = torch.nn.functional.normalize(u + qq, p=2, dim=1, eps=1e-6).detach()
        e = xc.unsqueeze(1)
        emb_out = (e - 2 * (e @ w.unsqueeze(-1) @ w.unsqueeze(1)) + 2 * (e @ u.unsqueeze(-1).detach() @ qq.unsqueeze(1).detach())).squeeze()
    loss = ((xc.detach() - emb) ** 2).sum(-1) + 0.25 * ((xc - emb.detach()) ** 2).sum(-1)
    (emb_out.sum() + loss.sum()).backward()
    torch.testing.assert_close(out.embeddings.detach().cpu(), emb_out.detach(), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(out.loss.detach().cpu(), loss.detach(), rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(x.grad.cpu(), xc.grad, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(q.embedding.weight.grad.cpu(), cb.grad, rtol=1e-4, atol=1e-5)
