"""Drop-in mirror of ``genrec.models.rqvae`` (reference: genrec/models/rqvae.py): semantic ids and training.

Semantic ids (SURVEY.md section 8 rows a10/a11): ``Quantize.forward`` in eval mode (distance + first-min argmin + codebook gather +
quantize loss, rqvae.py:185-199, :246-254) and the residual loop of ``RqVae.get_semantic_ids`` (:386-412), both executed by ONE launch of
the sm_90a kernel ``rq_residual_argmin`` (csrc/rq_argmin.cuh) for all levels.

Training (row f3): ``RqVae.forward(batch, gumbel_t)`` returns the reference's ``RqVaeComputedLosses`` (rqvae.py:414-454) in train and
eval mode.  The SINKHORN estimator's 100 fp64 Sinkhorn-Knopp iterations and its hard assignment are one launch of ``rq_sinkhorn``
(csrc/rq_sinkhorn.cuh); the k-means codebook initialisation (modules/kmeans.py) runs on the device, with the Lloyd update in
``kmeans_update_kernel`` and the assignment in ``rq_residual_argmin``.  STE, ROTATION_TRICK and GUMBEL_SOFTMAX keep the reference's
element-wise formulas around the kernel's nearest-code search, and the bias-free SiLU MLP encoder / decoder (encoder.py:380-420) train on
torch's fp32 cuBLAS GEMMs.
Out of scope (raise): fusing the GUMBEL_SOFTMAX estimator, cosine distance, ``sim_vq`` and ``codebook_normalize``.
"""
from __future__ import annotations

from enum import Enum
from typing import List, NamedTuple

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import functional as Fn
from ._lib import ensure_device, require_cuda


class QuantizeForwardMode(Enum):
    GUMBEL_SOFTMAX = 1
    STE = 2
    ROTATION_TRICK = 3
    SINKHORN = 4


class QuantizeDistance(Enum):
    L2 = 1
    COSINE = 2


class QuantizeOutput(NamedTuple):
    embeddings: torch.Tensor
    ids: torch.Tensor
    loss: torch.Tensor


class RqVaeOutput(NamedTuple):
    embeddings: torch.Tensor
    residuals: torch.Tensor
    sem_ids: torch.Tensor
    quantize_loss: torch.Tensor


class RqVaeComputedLosses(NamedTuple):
    loss: torch.Tensor
    reconstruction_loss: torch.Tensor
    rqvae_loss: torch.Tensor
    embs_norm: torch.Tensor
    p_unique_ids: torch.Tensor


class L2Norm(nn.Module):
    """genrec/modules/normalize.py:10-33: F.normalize(x, p=2, dim, eps); no parameters."""

    def __init__(self, dim: int = -1, eps: float = 1e-12) -> None:
        super().__init__()
        self.dim, self.eps = dim, eps

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return F.normalize(x, p=2, dim=self.dim, eps=self.eps)


class MLP(nn.Module):
    """Mirror of genrec/modules/encoder.py:380-420 (bias-free Linear + SiLU stack, then L2Norm or Identity; keys
    ``mlp.{0,2,4,...}.weight``)."""

    def __init__(self, input_dim: int, hidden_dims: List[int], out_dim: int, dropout: float = 0.0, normalize: bool = False):
        super().__init__()
        assert dropout == 0.0, "only the configuration shipped by the reference configs is mirrored"
        self.input_dim, self.hidden_dims, self.out_dim, self.normalize = input_dim, hidden_dims, out_dim, normalize
        dims = [input_dim] + list(hidden_dims) + [out_dim]
        self.mlp = nn.Sequential()
        for i, (a, b) in enumerate(zip(dims[:-1], dims[1:])):
            self.mlp.append(nn.Linear(a, b, bias=False))
            if i != len(dims) - 2:
                self.mlp.append(nn.SiLU())
        self.mlp.append(L2Norm() if normalize else nn.Identity())

    def _split_weights(self):
        """bf16 three-term splits of the layer weights (weight layout of the fp32-accurate GEMM), cached per parameter version."""
        lins = [m for m in self.mlp if isinstance(m, nn.Linear)]
        key = tuple((w.weight._version, w.weight.data_ptr()) for w in lins)
        if getattr(self, "_split_key", None) != key:
            self._split = [Fn.split3(w.weight, 1) for w in lins]
            self._split_key = key
        return self._split

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        assert x.shape[-1] == self.input_dim, f"Invalid input dim: Expected {self.input_dim}, found {x.shape[-1]}"
        if x.is_cuda and not (torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters()))):
            # inference (get_semantic_ids): every layer is one wgmma GEMM on three-term bf16 splits of both operands with the
            # SiLU in its epilogue - fp32 accuracy (the semantic ids must not depend on a bf16 rounding of the latent)
            ws = self._split_weights()
            h = x.detach().float().contiguous()
            for i, w in enumerate(ws):
                h = Fn.linear_f32x3(Fn.split3(h, 0), w, act=1 if i != len(ws) - 1 else 0)
            return F.normalize(h, p=2, dim=-1, eps=1e-12) if self.normalize else h
        return self.mlp(x)     # training of the encoder (autograd) stays on the library GEMM: out of scope of the hot path


SINKHORN_EPS, SINKHORN_ITERS = 0.003, 100        # rqvae.py:229-235
KMEANS_STOP, KMEANS_MAX_ITERS = 1e-10, 10_000


@torch.no_grad()
def kmeans_init_(weight: torch.Tensor, x: torch.Tensor, stop_threshold: float = KMEANS_STOP, max_iters: int = KMEANS_MAX_ITERS) -> int:
    """Lloyd's k-means of genrec/modules/kmeans.py:11-99 on the device; writes the centroids into ``weight`` [k, D] and returns the
    index of the converging iteration.  The same RNG use as the reference: the initial rows from ``np.random.choice(B, k,
    replace=False)``, and one ``torch.randint(0, B, (1,))`` draw of the CPU generator per empty cluster, in ascending cluster order.
    Each iteration is the nearest-centroid search (``rq_residual_argmin``, first index on ties), the centroid update
    (``kmeans_update_kernel``) and one host read of the cluster sizes and shifts.  It stops when the largest centroid shift falls
    below ``stop_threshold``.  The reference has no cap, and on inputs with fewer than k distinct rows an empty cluster is reseeded
    at random forever: this raises after ``max_iters`` iterations instead."""
    require_cuda(x)
    ensure_device(x.device)
    k = weight.shape[0]
    x = x.detach().float().contiguous()
    B = x.shape[0]
    if B < k:
        raise ValueError(f"k-means needs at least k = {k} rows to draw its initial centroids from, got {B}")
    c = x[torch.from_numpy(np.random.choice(B, k, replace=False)).to(x.device)].contiguous()     # kmeans.py:52-56
    for it in range(max_iters):
        assign = Fn.rq_residual_argmin(x, c.unsqueeze(0), want_aux=False)[0][:, 0]                 # kmeans.py:59-62
        stats = Fn.kmeans_update(x, assign, c).cpu()                                              # kmeans.py:67-75
        counts, shift = stats[0], stats[1].view(torch.float32)
        full = counts > 0
        moved = float(shift[full].max()) if bool(full.any()) else 0.0
        empty = torch.nonzero(~full).flatten()
        if len(empty):                                                                            # kmeans.py:69-73
            rows = torch.cat([torch.randint(0, B, (1,)) for _ in range(len(empty))]).to(x.device)
            empty = empty.to(x.device)
            if moved < stop_threshold:       # only then can the reseeded clusters decide whether this was the last iteration
                moved = max(moved, float(torch.linalg.vector_norm(x[rows] - c[empty], dim=1).max()))
            c[empty] = x[rows]
        if moved < stop_threshold:                                                                # kmeans.py:92-93
            weight.data.copy_(c)
            return it
    raise RuntimeError(f"k-means did not converge in {max_iters} iterations (B = {B}, k = {k}): with fewer than k distinct rows some "
                       "cluster stays empty and is reseeded at random every iteration")


def p_unique_ids(sem_ids: torch.Tensor, codebook_size: int) -> torch.Tensor:
    """Fraction of rows whose semantic id differs from every later row's, i.e. distinct ids / B (rqvae.py:443-446), without the
    [B, B, levels] comparison and without a host synchronisation: the ids of a row are packed into one int64 key and sorted."""
    B, levels = sem_ids.shape
    bits = max(1, (codebook_size - 1).bit_length())
    if levels * bits > 63:
        raise NotImplementedError(f"p_unique_ids packs {levels} levels x {bits} bits into an int64 key; at most 63 bits are supported")
    key = (sem_ids << (torch.arange(levels, device=sem_ids.device) * bits)).sum(-1)
    key = key.sort().values
    return (1 + (key[1:] != key[:-1]).sum()) / B


def _rotation_trick(u: torch.Tensor, q: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """genrec/models/rqvae.py:67-83 (efficient_rotation_trick_transform): rotate e from direction u onto direction q without
    forming the rotation matrix; u, q unit vectors [N, D], gradients flow through e only."""
    e = e.unsqueeze(1)                                            # [N, 1, D]
    w = F.normalize(u + q, p=2, dim=1, eps=1e-6).detach()
    return (e - 2 * (e @ w.unsqueeze(-1) @ w.unsqueeze(1)) + 2 * (e @ u.unsqueeze(-1).detach() @ q.unsqueeze(1).detach())).squeeze()


class Quantize(nn.Module):
    """Mirror of genrec/models/rqvae.py:115-254 (L2 distance, out_proj = Identity).  The k-means initialisation runs in
    ``RqVae.forward``; every reference caller of a standalone Quantize builds it without."""

    def __init__(self, embed_dim: int, n_embed: int, do_kmeans_init: bool = True, codebook_normalize: bool = False,
                 sim_vq: bool = False, commitment_weight: float = 0.25,
                 forward_mode: QuantizeForwardMode = QuantizeForwardMode.GUMBEL_SOFTMAX,
                 distance_mode: QuantizeDistance = QuantizeDistance.L2) -> None:
        super().__init__()
        if codebook_normalize or sim_vq or distance_mode != QuantizeDistance.L2:
            raise NotImplementedError("genrec_b200 mirrors the shipped configuration: L2 distance, out_proj = Identity")
        self.embed_dim, self.n_embed = embed_dim, n_embed
        self.embedding = nn.Embedding(n_embed, embed_dim)
        self.forward_mode, self.distance_mode = forward_mode, distance_mode
        self.do_kmeans_init = do_kmeans_init
        self.kmeans_initted = False
        self.commitment_weight = commitment_weight
        nn.init.uniform_(self.embedding.weight)     # rqvae.py:160-163

    @property
    def weight(self) -> torch.Tensor:
        return self.embedding.weight

    @property
    def device(self) -> torch.device:
        return self.embedding.weight.device

    def get_item_embeddings(self, item_ids) -> torch.Tensor:
        return self.embedding(item_ids)

    def forward(self, x: torch.Tensor, temperature=None) -> QuantizeOutput:
        assert x.shape[-1] == self.embed_dim
        require_cuda(x)
        ensure_device(x.device)
        if not self.training:
            ids, emb, _res, loss = Fn.rq_residual_argmin(x, self.embedding.weight.unsqueeze(0), self.commitment_weight)
            return QuantizeOutput(embeddings=emb[:, :, 0], ids=ids[:, 0], loss=loss)
        # training (rqvae.py:201-245): the nearest-code search (STE, rotation trick) or the Sinkhorn assignment is a CUDA kernel (ids
        # are not differentiated, `dist.detach()` at rqvae.py:199); the estimator around it is the reference's element-wise formula
        codebook = self.embedding.weight
        if self.forward_mode == QuantizeForwardMode.SINKHORN:                                # rqvae.py:218-241
            with torch.no_grad():
                dist = (x ** 2).sum(1, keepdim=True) + (codebook.T ** 2).sum(0, keepdim=True) - 2 * x @ codebook.T
            ids = Fn.rq_sinkhorn(dist, SINKHORN_EPS, SINKHORN_ITERS)[0]
            emb = self.get_item_embeddings(ids)
            emb_out = x + (emb - x).detach()
        elif self.forward_mode == QuantizeForwardMode.GUMBEL_SOFTMAX:                        # rqvae.py:201-206
            ids = Fn.rq_residual_argmin(x, codebook.unsqueeze(0), self.commitment_weight, want_aux=False)[0][:, 0]
            dist = (x ** 2).sum(1, keepdim=True) + (codebook.T ** 2).sum(0, keepdim=True) - 2 * x @ codebook.T
            u = torch.rand(dist.shape, device=x.device)
            y = -dist + -torch.log(-torch.log(u + 1e-20) + 1e-20)                            # modules/gumbel.py:10-46
            emb = F.softmax(y / temperature, dim=-1) @ codebook
            emb_out = emb
        else:
            ids = Fn.rq_residual_argmin(x, codebook.unsqueeze(0), self.commitment_weight, want_aux=False)[0][:, 0]
            emb = self.get_item_embeddings(ids)
            if self.forward_mode == QuantizeForwardMode.STE:                                 # rqvae.py:207-209
                emb_out = x + (emb - x).detach()
            else:                                                                            # rqvae.py:210-216
                emb_out = _rotation_trick(x / (x.norm(dim=-1, keepdim=True) + 1e-8), emb / (emb.norm(dim=-1, keepdim=True) + 1e-8), x)
        emb_loss = ((x.detach() - emb) ** 2).sum(-1)                                          # modules/loss.py:75-77
        query_loss = ((x - emb.detach()) ** 2).sum(-1)
        return QuantizeOutput(embeddings=emb_out, ids=ids, loss=emb_loss + self.commitment_weight * query_loss)


class RqVae(nn.Module):
    """Mirror of genrec/models/rqvae.py:277-454."""

    def __init__(self, input_dim: int, embed_dim: int, hidden_dims: List[int], codebook_size: int,
                 codebook_kmeans_init: bool = True, codebook_normalize: bool = False, codebook_sim_vq: bool = False,
                 codebook_mode: QuantizeForwardMode = QuantizeForwardMode.GUMBEL_SOFTMAX,
                 codebook_last_layer_mode: QuantizeForwardMode = QuantizeForwardMode.GUMBEL_SOFTMAX, n_layers: int = 3,
                 commitment_weight: float = 0.25, n_cat_features: int = 18) -> None:
        super().__init__()
        self._config = dict(input_dim=input_dim, embed_dim=embed_dim, hidden_dims=hidden_dims, codebook_size=codebook_size,
                            codebook_kmeans_init=codebook_kmeans_init, codebook_normalize=codebook_normalize,
                            codebook_sim_vq=codebook_sim_vq, codebook_mode=codebook_mode, codebook_last_layer_mode=codebook_last_layer_mode,
                            n_layers=n_layers, commitment_weight=commitment_weight, n_cat_features=n_cat_features)
        self.input_dim, self.embed_dim, self.hidden_dims = input_dim, embed_dim, hidden_dims
        self.n_layers, self.codebook_size, self.commitment_weight = n_layers, codebook_size, commitment_weight
        self.n_cat_feats = n_cat_features
        self.layers = nn.ModuleList([
            Quantize(embed_dim=embed_dim, n_embed=codebook_size,
                     forward_mode=codebook_mode if i < n_layers - 1 else codebook_last_layer_mode,
                     do_kmeans_init=codebook_kmeans_init, codebook_normalize=(i == 0 and codebook_normalize),
                     sim_vq=codebook_sim_vq, commitment_weight=commitment_weight) for i in range(n_layers)])
        self.encoder = MLP(input_dim=input_dim, hidden_dims=hidden_dims, out_dim=embed_dim)
        self.decoder = MLP(input_dim=embed_dim, hidden_dims=hidden_dims[-1::-1], out_dim=input_dim, normalize=True)

    @property
    def config(self) -> dict:
        """The constructor arguments (saved by the reference trainer as ``model_config``)."""
        return dict(self._config)

    @property
    def device(self) -> torch.device:
        return next(self.encoder.parameters()).device

    def load_pretrained(self, path: str) -> None:
        state = torch.load(path, map_location=self.device, weights_only=False)
        self.load_state_dict(state["model"])

    def encode(self, x: torch.Tensor) -> torch.Tensor:
        return self.encoder(x)

    def decode(self, x: torch.Tensor) -> torch.Tensor:
        return self.decoder(x)

    def codebooks(self) -> torch.Tensor:
        return torch.stack([l.embedding.weight for l in self.layers])     # [levels, K, D]

    @torch.no_grad()
    def get_semantic_ids(self, x: torch.Tensor, gumbel_t: float = 0.001) -> RqVaeOutput:
        """rqvae.py:386-412: encoder, then all residual levels in one kernel launch."""
        require_cuda(x)
        ensure_device(x.device)
        res = self.encode(x)
        ids, emb, residuals, loss = Fn.rq_residual_argmin(res, self.codebooks(), self.commitment_weight)
        return RqVaeOutput(embeddings=emb, residuals=residuals, sem_ids=ids, quantize_loss=loss)

    def forward(self, batch: torch.Tensor, gumbel_t: float) -> RqVaeComputedLosses:
        """rqvae.py:414-454 in train or eval mode.  On the first call every level with ``do_kmeans_init`` set initialises its codebook
        by k-means on its input residual before it quantises (rqvae.py:182-183)."""
        require_cuda(batch)
        ensure_device(batch.device)
        x = batch
        res = self.encode(x)
        quantize_loss = 0
        embs, sem_ids = [], []
        for layer in self.layers:
            if layer.do_kmeans_init and not layer.kmeans_initted:
                kmeans_init_(layer.embedding.weight, res)
                layer.kmeans_initted = True
            q = layer(res, temperature=gumbel_t)
            quantize_loss = quantize_loss + q.loss
            res = res - q.embeddings
            embs.append(q.embeddings)
            sem_ids.append(q.ids)
        embs = torch.stack(embs, -1)                                   # [B, D, levels]
        x_hat = self.decode(embs.sum(-1))
        n = self.n_cat_feats
        if n > 0:                                                      # modules/loss.py:26-54
            x_hat = torch.cat([F.normalize(x_hat[..., :-n], p=2, dim=-1, eps=1e-12), x_hat[..., -n:]], dim=-1)
            rec = ((x_hat[:, :-n] - x[:, :-n]) ** 2).sum(-1)
            rec = rec + F.binary_cross_entropy_with_logits(x_hat[:, -n:], x[:, -n:], reduction="none").sum(-1)
        else:                                                          # modules/loss.py:8-23
            x_hat = F.normalize(x_hat, p=2, dim=-1, eps=1e-12)
            rec = ((x_hat - x) ** 2).sum(-1)
        with torch.no_grad():
            embs_norm = embs.norm(dim=1)
            p_unique = p_unique_ids(torch.stack(sem_ids, -1), self.codebook_size)
        return RqVaeComputedLosses(loss=(rec + quantize_loss).mean(), reconstruction_loss=rec.mean(), rqvae_loss=quantize_loss.mean(),
                                   embs_norm=embs_norm, p_unique_ids=p_unique)
