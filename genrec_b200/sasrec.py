"""Drop-in mirror of ``genrec.models.sasrec`` (reference: genrec/models/sasrec.py) on the sm_90a C-ABI library.

Same classes / constructor arguments / forward signatures / parameter names (SURVEY.md Appendix C).  The hot item of
this model - the causal softmax attention core (sasrec.py:206-240) - runs in the flash-style CUDA kernels of
csrc/attn_sasrec.cuh (forward + backward); the projections / FFN are the wgmma GEMMs with fused bias / ReLU / dropout /
residual / mask epilogues, LayerNorm and the embedding are our row kernels.  A handful of element-wise glue operations of
the block's backward (mask multiply, one bf16+fp32 add) are plain torch ops on CUDA tensors.  CPU tensors raise.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.nn as nn

from . import functional as Fn
from ._lib import ensure_device, require_cuda

SITE_ATT, SITE_HID, SITE_OUT = 3, 1, 2   # dropout sites inside one block (layer * 8 + site)


class _BlockFn(torch.autograd.Function):
    """One SASRecBlock (sasrec.py:152-165) + the optional trailing `x * mask` of SASRec.forward (:116)."""

    @staticmethod
    def forward(ctx, x, rowmask, pad, cfg, bf16w, *params):
        (g1, b1, wq, bq, wk, bk, wv, bv, g2, b2, w1, bb1, w2, bb2) = params
        H, layer, p, seed, sd, apply_mask = cfg["H"], cfg["layer"], cfg["p"], cfg["seed"], cfg["seed_dev"], cfg["apply_mask"]
        x = x.detach().contiguous().float()
        qb, qf, st1 = Fn.layernorm_fwd(x, g1.detach(), b1.detach(), 1e-8, want_bf16=True, want_f32=True)        # :160 norm1
        xb = Fn.cast_rows_bf16(x)
        Q, _ = Fn.linear_fwd(qb, bf16w["wq"], bq.detach(), 0)                                                    # :201-203
        K, _ = Fn.linear_fwd(xb, bf16w["wk"], bk.detach(), 0)
        V, _ = Fn.linear_fwd(xb, bf16w["wv"], bv.detach(), 0)
        att, lse = Fn.sasrec_attention_fwd(Q, K, V, pad, H, p, seed, sd, layer)                                   # :206-240
        h = att.float() + qf                                                                                      # :244 residual = normalised query
        hnb, _, st2 = Fn.layernorm_fwd(h, g2.detach(), b2.detach(), 1e-8)                                        # :163 norm2
        z1, a1 = Fn.linear_fwd(hnb, bf16w["w1"], bb1.detach(), 2, p, seed, sd, layer * 8 + SITE_HID)              # fc1 + relu + dropout
        y = Fn.linear_residual_fwd(a1, bf16w["w2"], bb2.detach(), h, rowmask if apply_mask else None, p, seed, sd,
                                   layer * 8 + SITE_OUT)                                                          # fc2 + dropout + residual (* mask)
        ctx.cfg, ctx.bf16w = cfg, bf16w
        ctx.save_for_backward(x, rowmask, pad, st1, st2, qb, xb, Q, K, V, att, lse, h, hnb, z1, a1, g1, g2)
        return y

    @staticmethod
    def backward(ctx, dy):
        cfg, w = ctx.cfg, ctx.bf16w
        H, layer, p, seed, sd, apply_mask = cfg["H"], cfg["layer"], cfg["p"], cfg["seed"], cfg["seed_dev"], cfg["apply_mask"]
        x, rowmask, pad, st1, st2, qb, xb, Q, K, V, att, lse, h, hnb, z1, a1, g1, g2 = ctx.saved_tensors
        dy = dy.contiguous().float()
        if apply_mask:
            dy = dy * rowmask.view(*dy.shape[:-1], 1)
        dyb = Fn.cast_rows_bf16(dy, None, p, seed, sd, layer * 8 + SITE_OUT)
        _, dw2, db2 = Fn.linear_bwd(dyb, w["w2"], a1, need_dx=False)
        dz1 = Fn.linear_dact_bwd(dyb, w["w2"], z1, 2, p, seed, sd, layer * 8 + SITE_HID)
        dhn, dw1, db1 = Fn.linear_bwd(dz1, w["w1"], hnb)
        dh, dg2, dbt2 = Fn.layernorm_bwd(dhn, h, st2, g2, residual=dy)
        datt = Fn.cast_rows_bf16(dh)
        dQ, dK, dV = Fn.sasrec_attention_bwd(Q, K, V, pad, att, lse, datt, H, p, seed, sd, layer)
        dq, dwq, dbq = Fn.linear_bwd(dQ, w["wq"], qb, dx_residual=dh)          # + residual path through the normalised query
        dxk, dwk, dbk = Fn.linear_bwd(dK, w["wk"], xb)
        dxkv, dwv, dbv = Fn.linear_bwd(dV, w["wv"], xb, dx_residual=dxk)
        dx, dg1, dbt1 = Fn.layernorm_bwd(dq, x, st1, g1, residual=dxkv)
        return (dx, None, None, None, None, dg1, dbt1, dwq, dbq, dwk, dbk, dwv, dbv, dg2, dbt2, dw1, db1, dw2, db2)


class MultiHeadAttention(nn.Module):
    """Mirror of genrec/models/sasrec.py:168-246 (stand-alone use; inside SASRecBlock the fused block path is taken)."""

    def __init__(self, embed_dim: int, num_heads: int, dropout: float):
        super().__init__()
        assert embed_dim % num_heads == 0
        self.embed_dim, self.num_heads, self.head_dim = embed_dim, num_heads, embed_dim // num_heads
        self.scale = self.head_dim ** -0.5
        self.q_proj = nn.Linear(embed_dim, embed_dim)
        self.k_proj = nn.Linear(embed_dim, embed_dim)
        self.v_proj = nn.Linear(embed_dim, embed_dim)
        self.dropout = nn.Dropout(dropout)

    def forward(self, query: torch.Tensor, key_value: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
        return _AttnFn.apply(query, key_value, mask, self.num_heads, self.dropout.p if self.training else 0.0,
                             self.q_proj.weight, self.q_proj.bias, self.k_proj.weight, self.k_proj.bias, self.v_proj.weight,
                             self.v_proj.bias)


class _AttnFn(torch.autograd.Function):
    """MultiHeadAttention.forward as a unit: projections + attention core + `+ query` residual."""

    @staticmethod
    def forward(ctx, query, key_value, mask, H, p, wq, bq, wk, bk, wv, bv):
        require_cuda(query, key_value)
        ensure_device(query.device)
        q = query.detach().contiguous().float()
        kv = key_value.detach().contiguous().float()
        pad = (mask.reshape(q.shape[0], q.shape[1]) == 0).to(torch.uint8).contiguous()
        wqb, wkb, wvb = Fn.cast_bf16(wq), Fn.cast_bf16(wk), Fn.cast_bf16(wv)
        qb, kvb = Fn.cast_rows_bf16(q), Fn.cast_rows_bf16(kv)
        Q, _ = Fn.linear_fwd(qb, wqb, bq.detach(), 0)
        K, _ = Fn.linear_fwd(kvb, wkb, bk.detach(), 0)
        V, _ = Fn.linear_fwd(kvb, wvb, bv.detach(), 0)
        seed = torch.initial_seed() & 0x7FFFFFFFFFFFFFFF if p > 0 else 0
        att, lse = Fn.sasrec_attention_fwd(Q, K, V, pad, H, p, seed, None, 0)
        ctx.save_for_backward(pad, qb, kvb, Q, K, V, att, lse, wqb, wkb, wvb)
        ctx.cfg = (H, p, seed)
        return att.float() + q

    @staticmethod
    def backward(ctx, dout):
        pad, qb, kvb, Q, K, V, att, lse, wqb, wkb, wvb = ctx.saved_tensors
        H, p, seed = ctx.cfg
        dout = dout.contiguous().float()
        dQ, dK, dV = Fn.sasrec_attention_bwd(Q, K, V, pad, att, lse, Fn.cast_rows_bf16(dout), H, p, seed, None, 0)
        dq, dwq, dbq = Fn.linear_bwd(dQ, wqb, qb, dx_residual=dout)
        dk, dwk, dbk = Fn.linear_bwd(dK, wkb, kvb)
        dkv, dwv, dbv = Fn.linear_bwd(dV, wvb, kvb, dx_residual=dk)
        return dq, dkv, None, None, None, dwq, dbq, dwk, dbk, dwv, dbv


class _FfnFn(torch.autograd.Function):
    """PointWiseFeedForward.forward as a unit (sasrec.py:258-266): fc1 + ReLU + dropout, fc2 + dropout + residual - the same two
    fused-epilogue GEMMs the block path runs."""

    @staticmethod
    def forward(ctx, x, residual, p, w1, b1, w2, b2):
        require_cuda(x, residual)
        ensure_device(x.device)
        xf = x.detach().contiguous().float()
        res = residual.detach().contiguous().float()
        w1b, w2b = Fn.cast_bf16(w1), Fn.cast_bf16(w2)
        xb = Fn.cast_rows_bf16(xf)
        seed = torch.initial_seed() & 0x7FFFFFFFFFFFFFFF if p > 0 else 0
        z1, a1 = Fn.linear_fwd(xb, w1b, b1.detach(), 2, p, seed, None, SITE_HID)
        y = Fn.linear_residual_fwd(a1, w2b, b2.detach(), res, None, p, seed, None, SITE_OUT)
        ctx.save_for_backward(xb, z1, a1, w1b, w2b)
        ctx.cfg = (p, seed)
        return y

    @staticmethod
    def backward(ctx, dy):
        xb, z1, a1, w1b, w2b = ctx.saved_tensors
        p, seed = ctx.cfg
        dy = dy.contiguous().float()
        dyb = Fn.cast_rows_bf16(dy, None, p, seed, None, SITE_OUT)
        _, dw2, db2 = Fn.linear_bwd(dyb, w2b, a1, need_dx=False)
        dz1 = Fn.linear_dact_bwd(dyb, w2b, z1, 2, p, seed, None, SITE_HID)
        dx, dw1, db1 = Fn.linear_bwd(dz1, w1b, xb)
        return dx, dy, None, dw1, db1, dw2, db2


class PointWiseFeedForward(nn.Module):
    """Mirror of genrec/models/sasrec.py:249-266.  Inside a SASRecBlock the fused block path runs it; called on its own it is the
    same pair of kernels behind an autograd function."""

    def __init__(self, embed_dim: int, ffn_dim: int, dropout: float):
        super().__init__()
        self.fc1 = nn.Linear(embed_dim, ffn_dim)
        self.fc2 = nn.Linear(ffn_dim, embed_dim)
        self.dropout = nn.Dropout(dropout)

    def forward(self, x: torch.Tensor, residual: torch.Tensor) -> torch.Tensor:
        """x: normalised input [B, L, D]; residual: the block input [B, L, D]  ->  fc2(drop(relu(fc1(x)))) dropped + residual."""
        return _FfnFn.apply(x, residual, self.dropout.p if self.training else 0.0, self.fc1.weight, self.fc1.bias, self.fc2.weight,
                            self.fc2.bias)


class SASRecBlock(nn.Module):
    """Mirror of genrec/models/sasrec.py:141-165."""

    def __init__(self, embed_dim: int, num_heads: int, ffn_dim: int, dropout: float):
        super().__init__()
        self.attention = MultiHeadAttention(embed_dim, num_heads, dropout)
        self.ffn = PointWiseFeedForward(embed_dim, ffn_dim, dropout)
        self.norm1 = nn.LayerNorm(embed_dim, eps=1e-8)
        self.norm2 = nn.LayerNorm(embed_dim, eps=1e-8)
        self.layer_index = 0
        self.p = dropout

    def _params(self):
        a, f = self.attention, self.ffn
        return (self.norm1.weight, self.norm1.bias, a.q_proj.weight, a.q_proj.bias, a.k_proj.weight, a.k_proj.bias, a.v_proj.weight,
                a.v_proj.bias, self.norm2.weight, self.norm2.bias, f.fc1.weight, f.fc1.bias, f.fc2.weight, f.fc2.bias)

    def forward(self, x: torch.Tensor, mask: torch.Tensor, _apply_mask: bool = False, _seed: int = 0, _seed_dev=None) -> torch.Tensor:
        """x [B,L,D] fp32, mask [B,L,1] float (1 = valid)."""
        require_cuda(x)
        ensure_device(x.device)
        B, L, _ = x.shape
        rowmask = mask.reshape(B * L).float().contiguous()
        pad = (rowmask == 0).to(torch.uint8).view(B, L).contiguous()
        a, f = self.attention, self.ffn
        bf16w = dict(wq=Fn.cast_bf16(a.q_proj.weight), wk=Fn.cast_bf16(a.k_proj.weight), wv=Fn.cast_bf16(a.v_proj.weight),
                     w1=Fn.cast_bf16(f.fc1.weight), w2=Fn.cast_bf16(f.fc2.weight))
        cfg = dict(H=a.num_heads, layer=self.layer_index, p=self.p if self.training else 0.0, seed=_seed, seed_dev=_seed_dev,
                   apply_mask=_apply_mask)
        return _BlockFn.apply(x, rowmask, pad, cfg, bf16w, *self._params())


class SASRec(nn.Module):
    """Mirror of genrec/models/sasrec.py:18-138."""

    def __init__(self, num_items: int, max_seq_len: int = 50, embed_dim: int = 64, num_heads: int = 2, num_blocks: int = 2,
                 ffn_dim: int = 256, dropout: float = 0.2):
        super().__init__()
        self.num_items, self.max_seq_len, self.embed_dim = num_items, max_seq_len, embed_dim
        self.item_embedding = nn.Embedding(num_items + 1, embed_dim, padding_idx=0)
        self.position_embedding = nn.Embedding(max_seq_len, embed_dim)
        self.emb_dropout = nn.Dropout(dropout)
        self.blocks = nn.ModuleList([SASRecBlock(embed_dim, num_heads, ffn_dim, dropout) for _ in range(num_blocks)])
        for i, b in enumerate(self.blocks):
            b.layer_index = i
        self.final_norm = nn.LayerNorm(embed_dim, eps=1e-8)
        self.return_train_logits = False
        self._seed_dev = None
        self._step_seed = 0
        self._init_weights()

    def _init_weights(self):
        """genrec/models/sasrec.py:64-77."""
        for module in self.modules():
            if isinstance(module, nn.Linear):
                nn.init.xavier_uniform_(module.weight)
                if module.bias is not None:
                    nn.init.zeros_(module.bias)
            elif isinstance(module, nn.Embedding):
                nn.init.xavier_uniform_(module.weight)
                if module.padding_idx is not None:
                    module.weight.data[module.padding_idx].zero_()
            elif isinstance(module, nn.LayerNorm):
                nn.init.ones_(module.weight)
                nn.init.zeros_(module.bias)

    def _seeds(self, device):
        if not (self.training and self.emb_dropout.p > 0):
            return 0, None
        if self._seed_dev is None or self._seed_dev.device != device:
            self._seed_dev = torch.zeros(1, dtype=torch.int64, device=device)
            self._step_seed = torch.initial_seed() & 0x7FFFFFFFFFFFFFFF
        self._seed_dev.add_(0x9E3779B1)
        # per-forward snapshot: the backward re-derives the masks from the value THIS forward saw
        return self._step_seed, self._seed_dev.clone()

    def forward(self, input_ids: torch.Tensor, targets: Optional[torch.Tensor] = None
                ) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """sasrec.py:79-130.  Returns (logits [B,L,V+1] fp32 | None when training with targets, loss | None)."""
        require_cuda(input_ids)
        ensure_device(input_ids.device)
        B, L = input_ids.shape
        assert L <= self.max_seq_len, "sequence longer than the position table"
        seed, sd = self._seeds(input_ids.device)
        p = self.emb_dropout.p if self.training else 0.0
        x, pad = Fn.EmbedFn.apply(input_ids, self.item_embedding.weight, self.position_embedding.weight, self.embed_dim ** 0.5, 1, p,
                                  seed, sd)                                                      # :100-111
        mask = (pad == 0).float().unsqueeze(-1)
        for blk in self.blocks:
            x = blk(x, mask, _apply_mask=True, _seed=seed, _seed_dev=sd)                         # :114-116
        table = self.item_embedding.weight
        table_bf16 = Fn.cast_bf16(table)
        logits = loss = None
        if targets is not None:
            loss = Fn.HeadLossFn.apply(x, self.final_norm.weight, self.final_norm.bias, table, table_bf16, targets, self.final_norm.eps)
        if targets is None or not self.training or self.return_train_logits:
            logits = Fn.head_logits(x, self.final_norm.weight, self.final_norm.bias, table, table_bf16, self.final_norm.eps)
        return logits, loss

    @torch.no_grad()
    def predict(self, input_ids: torch.Tensor, top_k: int = 10) -> torch.Tensor:
        """sasrec.py:132-138."""
        logits, _ = self.forward(input_ids)
        last_logits = logits[:, -1, :]
        last_logits[:, 0] = float("-inf")
        _, top_k_items = torch.topk(last_logits, top_k, dim=-1)
        return top_k_items
