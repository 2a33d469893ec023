"""Restatement of the RQ-VAE training path of the reference (genrec/models/rqvae.py:85-110, :165-254, :414-454;
genrec/modules/kmeans.py; genrec/modules/loss.py), written fresh in plain torch: the yardstick of test_rqvae_train_*.py.

Sinkhorn runs in fp64 with the reference's exact sequence of operations.  The reference's eager ``_sinkhorn_knopp`` multiplies the
fp64 kernel matrix with its fp32 ``v = ones`` and raises a dtype error; its ``forward`` only runs under ``torch.compile``, which
promotes that product to fp64.  This restatement starts from fp64 ``v = 1``, which is what the compiled graph computes.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn.functional as F

EPS, ITERS = 0.003, 100


def normalise(dist: torch.Tensor, rowwise: bool = False) -> torch.Tensor:
    """rqvae.py:221-224 in fp32, then widened to fp64 (``rowwise`` is a deliberate mistake for the mutation tests)."""
    if rowwise:
        mx, mn = dist.max(1, keepdim=True).values, dist.min(1, keepdim=True).values
    else:
        mx, mn = dist.max(), dist.min()
    mid = (mx + mn) / 2
    amp = mx - mid + 1e-5
    return ((dist - mid) / amp).double()


def sinkhorn(dist: torch.Tensor, eps: float = EPS, iters: int = ITERS, fp32_marginals: bool = True, swap: bool = False,
             rowwise: bool = False, stab: float = 1e-8):
    """dist [B, K] fp32 -> (ids [B], u [B], v [K], P [B, K]).  rqvae.py:85-110, :220-238.  The keyword arguments other than eps and
    iters only exist to restate deliberate mistakes."""
    B, K = dist.shape
    Km = torch.exp(-normalise(dist, rowwise) / eps)
    dev = dist.device
    if fp32_marginals:
        r = torch.full((B,), 1.0 / B, dtype=torch.float32, device=dev).double()
        c = torch.full((K,), 1.0 / K, dtype=torch.float32, device=dev).double()
    else:
        r = torch.full((B,), 1.0 / B, dtype=torch.float64, device=dev)
        c = torch.full((K,), 1.0 / K, dtype=torch.float64, device=dev)
    u = torch.ones(B, dtype=torch.float64, device=dev)
    v = torch.ones(K, dtype=torch.float64, device=dev)
    for _ in range(iters):
        if swap:
            v = c / (Km.T @ u + stab)
            u = r / (Km @ v + stab)
        else:
            u = r / (Km @ v + stab)
            v = c / (Km.T @ u + stab)
    P = u.unsqueeze(1) * Km * v.unsqueeze(0)
    return P.argmax(-1), u, v, P


def l2_dist(x: torch.Tensor, codebook: torch.Tensor) -> torch.Tensor:
    """rqvae.py:187-191."""
    return (x ** 2).sum(1, keepdim=True) + (codebook.T ** 2).sum(0, keepdim=True) - 2 * x @ codebook.T


def kmeans(x: torch.Tensor, k: int, stop: float = 1e-10, max_iters: Optional[int] = None, chunk: int = 4096):
    """Lloyd's algorithm of genrec/modules/kmeans.py:52-99 with its RNG use: initial rows from np.random.choice, one
    torch.randint(0, B, (1,)) CPU draw per empty cluster in ascending order.  Returns (centroids, converging iteration, initial rows).
    The [B, k, D] squared differences of kmeans.py:59-62 are formed in row chunks (same values, bounded memory)."""
    B = x.shape[0]
    init = np.random.choice(B, k, replace=False)
    c = x[torch.from_numpy(init).to(x.device)].clone()
    i = 0
    while max_iters is None or i < max_iters:
        old = c.clone()
        idx = torch.cat([((xc[:, None, :] - c[None, :, :]) ** 2).sum(2).min(1).indices for xc in x.split(chunk)])
        for cl in range(k):
            m = idx == cl
            if not m.any():
                c[cl] = x[torch.randint(0, B, (1,))].squeeze(0)
            else:
                c[cl] = x[m].mean(0)
        if torch.norm(c - old, dim=1).max() < stop:
            break
        i += 1
    return c, i, init


def mlp(x: torch.Tensor, weights: List[torch.Tensor], normalize: bool) -> torch.Tensor:
    """genrec/modules/encoder.py:399-420: bias-free Linear + SiLU, then L2Norm (eps 1e-12) or nothing."""
    for i, w in enumerate(weights):
        x = x @ w.T
        if i != len(weights) - 1:
            x = F.silu(x)
    return F.normalize(x, p=2, dim=-1, eps=1e-12) if normalize else x


def _weights(p: Dict[str, torch.Tensor], prefix: str) -> List[torch.Tensor]:
    keys = sorted((k for k in p if k.startswith(prefix + ".mlp.")), key=lambda k: int(k.split(".")[2]))
    return [p[k] for k in keys]


def train_forward(p: Dict[str, torch.Tensor], x: torch.Tensor, modes: List[str], training: bool = True, commitment: float = 0.25,
                  n_cat: int = 0, ids: Optional[List[torch.Tensor]] = None, codebook_size: int = 256):
    """RqVae.forward (rqvae.py:414-454) from a state dict ``p``; ``modes`` per level, "STE" or "SINKHORN".  ``ids`` replaces the
    search's ids level by level (the ids are not differentiated, so gradients given the same ids are comparable).  Returns
    (dict of the five outputs, ids per level)."""
    res = mlp(x, _weights(p, "encoder"), False)
    qloss, embs, out_ids = 0, [], []
    for lv, mode in enumerate(modes):
        cb = p[f"layers.{lv}.embedding.weight"]
        with torch.no_grad():
            dist = l2_dist(res, cb)
        if ids is not None:
            idl = ids[lv]
        elif training and mode == "SINKHORN":
            idl = sinkhorn(dist.detach())[0]
        else:
            idl = dist.min(1).indices
        emb = cb[idl]
        emb_out = res + (emb - res).detach() if training else emb
        qloss = qloss + ((res.detach() - emb) ** 2).sum(-1) + commitment * ((res - emb.detach()) ** 2).sum(-1)
        res = res - emb_out
        embs.append(emb_out)
        out_ids.append(idl)
    embs = torch.stack(embs, -1)
    x_hat = mlp(embs.sum(-1), _weights(p, "decoder"), True)
    if n_cat > 0:
        x_hat = torch.cat([F.normalize(x_hat[..., :-n_cat], p=2, dim=-1, eps=1e-12), x_hat[..., -n_cat:]], -1)
        rec = ((x_hat[:, :-n_cat] - x[:, :-n_cat]) ** 2).sum(-1) + F.binary_cross_entropy_with_logits(
            x_hat[:, -n_cat:], x[:, -n_cat:], reduction="none").sum(-1)
    else:
        x_hat = F.normalize(x_hat, p=2, dim=-1, eps=1e-12)
        rec = ((x_hat - x) ** 2).sum(-1)
    sem = torch.stack(out_ids, -1)
    with torch.no_grad():
        same = (sem[:, None, :] == sem[None, :, :]).all(-1)                # rqvae.py:443-446, [B, B]
        p_unique = (~torch.triu(same, diagonal=1)).all(1).sum() / sem.shape[0]
    return dict(loss=(rec + qloss).mean(), reconstruction_loss=rec.mean(), rqvae_loss=qloss.mean(), embs_norm=embs.detach().norm(dim=1),
                p_unique_ids=p_unique), out_ids


def seeded_state(input_dim: int, hidden: List[int], D: int, levels: int, K: int, seed: int) -> Dict[str, torch.Tensor]:
    """A reproducible RqVae state dict (CPU generator): Linear weights ~ U(-1/sqrt(fan_in), 1/sqrt(fan_in)) like nn.Linear's default,
    codebooks ~ U(0, 1) scaled down level by level so that every level sees non-trivial residuals."""
    g = torch.Generator().manual_seed(seed)
    p = {}
    for pre, dims in (("encoder", [input_dim] + hidden + [D]), ("decoder", [D] + hidden[::-1] + [input_dim])):
        for i, (a, b) in enumerate(zip(dims[:-1], dims[1:])):
            p[f"{pre}.mlp.{2 * i}.weight"] = (torch.rand(b, a, generator=g) * 2 - 1) / a ** 0.5
    for lv in range(levels):
        p[f"layers.{lv}.embedding.weight"] = (torch.rand(K, D, generator=g) - 0.5) * (0.5 / 2 ** lv)
    return p


def seeded_items(B: int, input_dim: int, seed: int, n_clusters: int = 64) -> torch.Tensor:
    """Unit-norm item vectors around ``n_clusters`` random centres (CPU generator)."""
    g = torch.Generator().manual_seed(seed)
    centres = torch.randn(n_clusters, input_dim, generator=g)
    x = centres[torch.randint(0, n_clusters, (B,), generator=g)] + 0.3 * torch.randn(B, input_dim, generator=g)
    return x / x.norm(dim=1, keepdim=True)
