"""Drop-in mirror of the RQ-VAE semantic-id path of ``genrec.models.rqvae`` (reference: genrec/models/rqvae.py).

In scope (SURVEY.md section 8 rows a10/a11): ``Quantize.forward`` in eval mode (distance + first-min argmin + codebook
gather + quantize loss, rqvae.py:185-199, :246-254) and the residual loop of ``RqVae.get_semantic_ids`` (:386-412), both
executed by ONE launch of the sm_90a kernel ``rq_residual_argmin`` (csrc/rq_argmin.cuh) for all levels.
Out of scope (raise): training-mode estimators (Gumbel / STE / rotation trick / Sinkhorn), k-means init, the decoder and
the reconstruction losses.  The bias-free SiLU MLP encoder in front of the argmin (encoder.py:380-420, "next" row f3) runs
on cuBLAS through ``torch.nn.functional.linear``.
"""
from __future__ import annotations

from enum import Enum
from typing import List, NamedTuple

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


class MLP(nn.Module):
    """Mirror of genrec/modules/encoder.py:380-420 (bias-free Linear + SiLU stack; keys ``mlp.{0,2,4,...}.weight``)."""

    def __init__(self, input_dim: int, hidden_dims: List[int], out_dim: int, dropout: float = 0.0, normalize: bool = False):
        super().__init__()
        assert dropout == 0.0 and not normalize, "only the configuration shipped by the reference configs is mirrored"
        self.input_dim, self.hidden_dims, self.out_dim = input_dim, hidden_dims, out_dim
        dims = [input_dim] + list(hidden_dims) + [out_dim]
        self.mlp = nn.Sequential()
        for i, (a, b) in enumerate(zip(dims[:-1], dims[1:])):
            self.mlp.append(nn.Linear(a, b, bias=False))
            if i != len(dims) - 2:
                self.mlp.append(nn.SiLU())
        self.mlp.append(nn.Identity())

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
            return h
        return self.mlp(x)     # training of the encoder (autograd) stays on the library GEMM: out of scope of the hot path


def _rotation_trick(u: torch.Tensor, q: torch.Tensor, e: torch.Tensor) -> torch.Tensor:
    """genrec/models/rqvae.py:67-83 (efficient_rotation_trick_transform): rotate e from direction u onto direction q without
    forming the rotation matrix; u, q unit vectors [N, D], gradients flow through e only."""
    e = e.unsqueeze(1)                                            # [N, 1, D]
    w = F.normalize(u + q, p=2, dim=1, eps=1e-6).detach()
    return (e - 2 * (e @ w.unsqueeze(-1) @ w.unsqueeze(1)) + 2 * (e @ u.unsqueeze(-1).detach() @ q.unsqueeze(1).detach())).squeeze()


class Quantize(nn.Module):
    """Mirror of genrec/models/rqvae.py:115-254 (eval-mode L2 path)."""

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
        # training (rqvae.py:201-245): the nearest-code search is the CUDA kernel (ids are not differentiated, `dist.detach()`
        # at rqvae.py:199); the estimator around it is the reference's element-wise formula on [N, D] tensors
        ids = Fn.rq_residual_argmin(x, self.embedding.weight.unsqueeze(0), self.commitment_weight, want_aux=False)[0][:, 0]
        codebook = self.embedding.weight
        if self.forward_mode == QuantizeForwardMode.STE:                                     # rqvae.py:207-209
            emb = self.get_item_embeddings(ids)
            emb_out = x + (emb - x).detach()
        elif self.forward_mode == QuantizeForwardMode.ROTATION_TRICK:                        # rqvae.py:210-216
            emb = self.get_item_embeddings(ids)
            emb_out = _rotation_trick(x / (x.norm(dim=-1, keepdim=True) + 1e-8), emb / (emb.norm(dim=-1, keepdim=True) + 1e-8), x)
        elif self.forward_mode == QuantizeForwardMode.GUMBEL_SOFTMAX:                        # rqvae.py:201-206
            dist = (x ** 2).sum(1, keepdim=True) + (codebook.T ** 2).sum(0, keepdim=True) - 2 * x @ codebook.T
            u = torch.rand(dist.shape, device=x.device)
            y = -dist + -torch.log(-torch.log(u + 1e-20) + 1e-20)                            # modules/gumbel.py:10-46
            emb = F.softmax(y / temperature, dim=-1) @ codebook
            emb_out = emb
        else:
            raise NotImplementedError("the Sinkhorn estimator (fp64, 100 iterations) is out of scope (SURVEY.md section 8, row f3)")
        emb_loss = ((x.detach() - emb) ** 2).sum(-1)                                          # modules/loss.py:75-77
        query_loss = ((x - emb.detach()) ** 2).sum(-1)
        return QuantizeOutput(embeddings=emb_out, ids=ids, loss=emb_loss + self.commitment_weight * query_loss)


class RqVae(nn.Module):
    """Mirror of genrec/models/rqvae.py:277-412 restricted to the semantic-id path."""

    def __init__(self, input_dim: int, embed_dim: int, hidden_dims: List[int], codebook_size: int,
                 codebook_kmeans_init: bool = True, codebook_normalize: bool = False, codebook_sim_vq: bool = False,
                 codebook_mode: QuantizeForwardMode = QuantizeForwardMode.GUMBEL_SOFTMAX,
                 codebook_last_layer_mode: QuantizeForwardMode = QuantizeForwardMode.GUMBEL_SOFTMAX, n_layers: int = 3,
                 commitment_weight: float = 0.25, n_cat_features: int = 18) -> None:
        super().__init__()
        self.input_dim, self.embed_dim, self.hidden_dims = input_dim, embed_dim, hidden_dims
        self.n_layers, self.codebook_size, self.commitment_weight = n_layers, codebook_size, commitment_weight
        self.n_cat_feats = n_cat_features
        self.layers = nn.ModuleList([
            Quantize(embed_dim=embed_dim, n_embed=codebook_size,
                     forward_mode=codebook_mode if i < n_layers - 1 else codebook_last_layer_mode,
                     do_kmeans_init=codebook_kmeans_init, codebook_normalize=(i == 0 and codebook_normalize),
                     sim_vq=codebook_sim_vq, commitment_weight=commitment_weight) for i in range(n_layers)])
        self.encoder = MLP(input_dim=input_dim, hidden_dims=hidden_dims, out_dim=embed_dim)
        # the decoder exists only so that reference checkpoints load with strict=True; it is never run here
        self.decoder = MLP(input_dim=embed_dim, hidden_dims=hidden_dims[-1::-1], out_dim=input_dim)

    @property
    def device(self) -> torch.device:
        return next(self.encoder.parameters()).device

    def load_pretrained(self, path: str) -> None:
        state = torch.load(path, map_location=self.device, weights_only=False)
        self.load_state_dict(state["model"])

    def encode(self, x: torch.Tensor) -> torch.Tensor:
        return self.encoder(x)

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

    def forward(self, batch, gumbel_t):
        raise NotImplementedError("RQ-VAE training (reconstruction + estimators) is out of scope; see SURVEY.md section 8")
