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
    """One SASRecBlock (sasrec.py:152-165) + the optional trailing `x * mask` of SASRec.forward (:116).  x [B, L, D] with pad [B, L],
    or a packed batch: x [T, D], rowmask / pad [T], and cfg["offsets"] ([B+1] on the device) with cfg["max_len"]."""

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
        att, lse = Fn.sasrec_attention_fwd(Q, K, V, pad, H, p, seed, sd, layer, cfg["offsets"], cfg["max_len"])   # :206-240
        h = att.float() + qf                                                                                      # :244 residual = normalised query
        hnb, _, st2 = Fn.layernorm_fwd(h, g2.detach(), b2.detach(), 1e-8)                                        # :163 norm2
        y, z1, a1 = Fn.ffn_fwd(hnb, bf16w["w1"], bb1.detach(), bf16w["w2"], bb2.detach(), h, rowmask if apply_mask else None, p, p,
                               seed, sd, layer * 8 + SITE_HID, layer * 8 + SITE_OUT)    # fc1 + relu + dropout, fc2 + dropout + residual (* mask)
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
        dhn, dw1, db1, dw2, db2 = Fn.ffn_bwd(dy, w["w1"], w["w2"], hnb, z1, a1, p, p, seed, sd, layer * 8 + SITE_HID,
                                             layer * 8 + SITE_OUT)
        dh, dg2, dbt2 = Fn.layernorm_bwd(dhn, h, st2, g2, residual=dy)
        datt = Fn.cast_rows_bf16(dh)
        dQ, dK, dV = Fn.sasrec_attention_bwd(Q, K, V, pad, att, lse, datt, H, p, seed, sd, layer, cfg["offsets"], cfg["max_len"])
        dq, dwq, dbq = Fn.linear_bwd(dQ, w["wq"], qb, dx_residual=dh)          # + residual path through the normalised query
        dxk, dwk, dbk = Fn.linear_bwd(dK, w["wk"], xb)
        dxkv, dwv, dbv = Fn.linear_bwd(dV, w["wv"], xb, dx_residual=dxk)
        dx, dg1, dbt1 = Fn.layernorm_bwd(dq, x, st1, g1, residual=dxkv)
        return (dx, None, None, None, None, dg1, dbt1, dwq, dbq, dwk, dbk, dwv, dbv, dg2, dbt2, dw1, db1, dw2, db2)


class MultiHeadAttention(Fn.StepSeeds, nn.Module):
    """Mirror of genrec/models/sasrec.py:168-246 (stand-alone use; inside SASRecBlock the fused block path is taken).  In training
    each call draws a fresh dropout mask (``StepSeeds``), as the reference's nn.Dropout does."""

    def __init__(self, embed_dim: int, num_heads: int, dropout: float):
        super().__init__()
        assert embed_dim % num_heads == 0
        self.embed_dim, self.num_heads, self.head_dim = embed_dim, num_heads, embed_dim // num_heads
        self.scale = self.head_dim ** -0.5
        self.q_proj = nn.Linear(embed_dim, embed_dim)
        self.k_proj = nn.Linear(embed_dim, embed_dim)
        self.v_proj = nn.Linear(embed_dim, embed_dim)
        self.dropout = nn.Dropout(dropout)

    @property
    def _dropout_p(self) -> float:
        return self.dropout.p

    def forward(self, query: torch.Tensor, key_value: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
        seed, sd = self._seeds(query.device)
        return _AttnFn.apply(query, key_value, mask, self.num_heads, self.dropout.p if self.training else 0.0, seed, sd,
                             self.q_proj.weight, self.q_proj.bias, self.k_proj.weight, self.k_proj.bias, self.v_proj.weight,
                             self.v_proj.bias)


class _AttnFn(torch.autograd.Function):
    """MultiHeadAttention.forward as a unit: projections + attention core + `+ query` residual; dropout at site 3 under (seed,
    seed_dev), the backward re-deriving the forward's mask from them."""

    @staticmethod
    def forward(ctx, query, key_value, mask, H, p, seed, sd, wq, bq, wk, bk, wv, bv):
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
        att, lse = Fn.sasrec_attention_fwd(Q, K, V, pad, H, p, seed, sd, 0)
        ctx.save_for_backward(pad, qb, kvb, Q, K, V, att, lse, wqb, wkb, wvb)
        ctx.cfg = (H, p, seed, sd)
        return att.float() + q

    @staticmethod
    def backward(ctx, dout):
        pad, qb, kvb, Q, K, V, att, lse, wqb, wkb, wvb = ctx.saved_tensors
        H, p, seed, sd = ctx.cfg
        dout = dout.contiguous().float()
        dQ, dK, dV = Fn.sasrec_attention_bwd(Q, K, V, pad, att, lse, Fn.cast_rows_bf16(dout), H, p, seed, sd, 0)
        dq, dwq, dbq = Fn.linear_bwd(dQ, wqb, qb, dx_residual=dout)
        dk, dwk, dbk = Fn.linear_bwd(dK, wkb, kvb)
        dkv, dwv, dbv = Fn.linear_bwd(dV, wvb, kvb, dx_residual=dk)
        return dq, dkv, None, None, None, None, None, dwq, dbq, dwk, dbk, dwv, dbv


class _FfnFn(torch.autograd.Function):
    """PointWiseFeedForward.forward as a unit (sasrec.py:258-266): fc1 + ReLU + dropout, fc2 + dropout + residual - the same two
    fused-epilogue GEMMs the block path runs, at sites 1 and 2 under (seed, seed_dev)."""

    @staticmethod
    def forward(ctx, x, residual, p, seed, sd, w1, b1, w2, b2):
        require_cuda(x, residual)
        ensure_device(x.device)
        xf = x.detach().contiguous().float()
        res = residual.detach().contiguous().float()
        w1b, w2b = Fn.cast_bf16(w1), Fn.cast_bf16(w2)
        xb = Fn.cast_rows_bf16(xf)
        y, z1, a1 = Fn.ffn_fwd(xb, w1b, b1.detach(), w2b, b2.detach(), res, None, p, p, seed, sd, SITE_HID, SITE_OUT)
        ctx.save_for_backward(xb, z1, a1, w1b, w2b)
        ctx.cfg = (p, seed, sd)
        return y

    @staticmethod
    def backward(ctx, dy):
        xb, z1, a1, w1b, w2b = ctx.saved_tensors
        p, seed, sd = ctx.cfg
        dy = dy.contiguous().float()
        dx, dw1, db1, dw2, db2 = Fn.ffn_bwd(dy, w1b, w2b, xb, z1, a1, p, p, seed, sd, SITE_HID, SITE_OUT)
        return dx, dy, None, None, None, dw1, db1, dw2, db2


class PointWiseFeedForward(Fn.StepSeeds, nn.Module):
    """Mirror of genrec/models/sasrec.py:249-266.  Inside a SASRecBlock the fused block path runs it; called on its own it is the
    same pair of kernels behind an autograd function, drawing a fresh dropout mask on each training call (``StepSeeds``)."""

    def __init__(self, embed_dim: int, ffn_dim: int, dropout: float):
        super().__init__()
        self.fc1 = nn.Linear(embed_dim, ffn_dim)
        self.fc2 = nn.Linear(ffn_dim, embed_dim)
        self.dropout = nn.Dropout(dropout)

    @property
    def _dropout_p(self) -> float:
        return self.dropout.p

    def forward(self, x: torch.Tensor, residual: torch.Tensor) -> torch.Tensor:
        """x: normalised input [B, L, D]; residual: the block input [B, L, D]  ->  fc2(drop(relu(fc1(x)))) dropped + residual."""
        seed, sd = self._seeds(x.device)
        return _FfnFn.apply(x, residual, self.dropout.p if self.training else 0.0, seed, sd, self.fc1.weight, self.fc1.bias,
                            self.fc2.weight, self.fc2.bias)


class SASRecBlock(Fn.StepSeeds, nn.Module):
    """Mirror of genrec/models/sasrec.py:141-165.  SASRec passes each block its step's seeds; called on its own without them, a
    training block draws fresh dropout masks on each call (``StepSeeds``)."""

    def __init__(self, embed_dim: int, num_heads: int, ffn_dim: int, dropout: float):
        super().__init__()
        self.attention = MultiHeadAttention(embed_dim, num_heads, dropout)
        self.ffn = PointWiseFeedForward(embed_dim, ffn_dim, dropout)
        self.norm1 = nn.LayerNorm(embed_dim, eps=1e-8)
        self.norm2 = nn.LayerNorm(embed_dim, eps=1e-8)
        self.layer_index = 0
        self.p = dropout

    @property
    def _dropout_p(self) -> float:
        return self.p

    def _params(self):
        a, f = self.attention, self.ffn
        return (self.norm1.weight, self.norm1.bias, a.q_proj.weight, a.q_proj.bias, a.k_proj.weight, a.k_proj.bias, a.v_proj.weight,
                a.v_proj.bias, self.norm2.weight, self.norm2.bias, f.fc1.weight, f.fc1.bias, f.fc2.weight, f.fc2.bias)

    def forward(self, x: torch.Tensor, mask: torch.Tensor, _apply_mask: bool = False, _seed: Optional[int] = None,
                _seed_dev=None) -> torch.Tensor:
        """x [B,L,D] fp32, mask [B,L,1] float (1 = valid).  _seed / _seed_dev: the step's seeds (SASRec passes them); None: the
        block's own."""
        require_cuda(x)
        ensure_device(x.device)
        if _seed is None:
            _seed, _seed_dev = self._seeds(x.device)
        B, L, _ = x.shape
        rowmask = mask.reshape(B * L).float().contiguous()
        pad = (rowmask == 0).to(torch.uint8).view(B, L).contiguous()
        return self._run(x, rowmask, pad, _apply_mask, _seed, _seed_dev)

    def _run(self, x, rowmask, pad, apply_mask, seed, seed_dev, offsets=None, max_len=None):
        a, f = self.attention, self.ffn
        bf16w = dict(wq=Fn.cast_bf16(a.q_proj.weight), wk=Fn.cast_bf16(a.k_proj.weight), wv=Fn.cast_bf16(a.v_proj.weight),
                     w1=Fn.cast_bf16(f.fc1.weight), w2=Fn.cast_bf16(f.fc2.weight))
        cfg = dict(H=a.num_heads, layer=self.layer_index, p=self.p if self.training else 0.0, seed=seed, seed_dev=seed_dev,
                   apply_mask=apply_mask, offsets=offsets, max_len=max_len)
        return _BlockFn.apply(x, rowmask, pad, cfg, bf16w, *self._params())


class SASRec(Fn.StepSeeds, nn.Module):
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
        self._init_weights()

    @property
    def _dropout_p(self) -> float:
        return self.emb_dropout.p

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

    def encode(self, input_ids: torch.Tensor) -> torch.Tensor:
        """Embedding + all blocks (everything before final_norm).  sasrec.py:100-116."""
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
        return x

    def forward(self, input_ids: torch.Tensor, targets: Optional[torch.Tensor] = None, *, negatives: Optional[torch.Tensor] = None,
                log_q: Optional[torch.Tensor] = None) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """sasrec.py:79-130.  Returns (logits [B,L,V+1] fp32 | None when training with targets, loss | None).  With ``negatives``
        ([N] int64, shared by every token) and optionally ``log_q`` ([V+1] fp32) the loss is the sampled softmax with logQ correction
        (see ``HSTU.forward``) and the result is ``(None, loss)``."""
        if negatives is None and log_q is not None:
            raise ValueError("log_q corrects the sampled softmax: pass negatives with it")
        if negatives is not None and targets is None:
            raise ValueError("negatives select the sampled-softmax loss, which needs targets")
        return self._head(self.encode(input_ids), targets, negatives, log_q)

    def _head(self, x: torch.Tensor, targets: Optional[torch.Tensor], negatives: Optional[torch.Tensor], log_q: Optional[torch.Tensor]
              ) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """The head of ``forward`` on x [B, L, D]: (logits [B, L, V+1] | None, loss | None) under forward's rules."""
        table = self.item_embedding.weight
        table_bf16 = Fn.cast_bf16(table)
        logits = loss = None
        if negatives is not None:
            return None, Fn.SampledHeadLossFn.apply(x, self.final_norm.weight, self.final_norm.bias, table, table_bf16, targets, negatives,
                                                    log_q, self.final_norm.eps)
        if targets is not None:
            loss = Fn.HeadLossFn.apply(x, self.final_norm.weight, self.final_norm.bias, table, table_bf16, targets, self.final_norm.eps)
        if targets is None or not self.training or self.return_train_logits:
            logits = Fn.head_logits(x, self.final_norm.weight, self.final_norm.bias, table, table_bf16, self.final_norm.eps)
        return logits, loss

    def encode_jagged(self, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int) -> torch.Tensor:
        """``encode`` of a packed batch: input_ids [T], offsets [B+1] int64 on the device (sequence b = rows offsets[b] ..
        offsets[b+1]-1), max_len >= every length (<= max_seq_len) -> [T, D] fp32.  Item i of a sequence of length n takes position
        P - n + i, P the batch's longest sequence (derived on the device), as in sasrec_collate_fn's left-padded batch."""
        T = input_ids.numel()
        seed, sd = self._seeds(input_ids.device)
        p = self.emb_dropout.p if self.training else 0.0
        x, pad = Fn.EmbedFn.apply(input_ids, self.item_embedding.weight, self.position_embedding.weight, self.embed_dim ** 0.5, 1, p,
                                  seed, sd, None, offsets, max_len)
        rowmask = (pad == 0).float()
        for blk in self.blocks:
            x = blk._run(x, rowmask, pad, True, seed, sd, offsets, max_len)
        return x.view(T, self.embed_dim)

    def forward_jagged(self, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int, targets: Optional[torch.Tensor] = None, *,
                       negatives: Optional[torch.Tensor] = None, log_q: Optional[torch.Tensor] = None
                       ) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """``forward`` on a packed batch (``data.pack_jagged``): input_ids / targets [T] int64, offsets [B+1] int64 (sequence b =
        rows offsets[b] .. offsets[b+1]-1; rows from offsets[B] to T are idle, id 0 and target 0), max_len >= every length and
        <= max_seq_len.  Returns (logits [T, V+1] fp32 | None, loss | None) under ``forward``'s rules (dropout, the sampled head,
        ``return_train_logits``).  Every stage runs on the T rows, none on padding.

        Position rule: item i of a sequence of length n sits at position P - n + i, P the longest sequence of the batch, as in the
        left-padded batch of sasrec_collate_fn; P is derived on the device, so every real token computes what it computes there
        (to fp32 summation order).  Dropout masks are keyed by token row, so under dropout a packed batch draws other masks.  With
        offsets on the CPU the batch is checked before any launch (ValueError); offsets on the device are not read on the host, so
        a step with fixed (B, T, max_len) can be captured in a CUDA graph and replayed with new offsets, ids and targets."""
        if negatives is None and log_q is not None:
            raise ValueError("log_q corrects the sampled softmax: pass negatives with it")
        if negatives is not None and targets is None:
            raise ValueError("negatives select the sampled-softmax loss, which needs targets")
        T = input_ids.numel()
        if targets is not None and tuple(targets.shape) != (T,):
            raise ValueError(f"forward_jagged: targets must be [{T}] like input_ids, got {tuple(targets.shape)}")
        offsets = Fn.check_jagged_batch("forward_jagged", input_ids, offsets, max_len, self.max_seq_len)   # the position table's rows
        x = self.encode_jagged(input_ids, offsets, max_len)
        logits, loss = self._head(x.view(1, T, self.embed_dim), targets.view(1, T) if targets is not None else None, negatives, log_q)
        return (logits.view(T, -1) if logits is not None else None), loss

    @torch.no_grad()
    def predict(self, input_ids: torch.Tensor, top_k: int = 10) -> torch.Tensor:
        """sasrec.py:132-138."""
        logits, _ = self.forward(input_ids)
        last_logits = logits[:, -1, :]
        last_logits[:, 0] = float("-inf")
        _, top_k_items = torch.topk(last_logits, top_k, dim=-1)
        return top_k_items

    @torch.no_grad()
    def recommend(self, input_ids: torch.Tensor, top_k: int = 10, exclude: Optional[torch.Tensor] = None) -> Fn.TopItems:
        """The ``top_k`` (1..64) best next items of each row as ``TopItems(scores, items)``, without forming the logits: the scores
        are bit-identical to the last row of ``forward``'s logits; item 0 and the row's ``exclude`` ids ([B, E] int64) never appear;
        equal scores go to the lower item id (see ``HSTU.recommend``)."""
        Fn.check_topk_args(top_k, exclude, input_ids.shape[0], input_ids.device)
        x = self.encode(input_ids)
        return Fn.head_topk(x[:, -1, :], self.final_norm.weight, self.final_norm.bias, Fn.cast_bf16(self.item_embedding.weight),
                            self.final_norm.eps, top_k, exclude)

    @torch.no_grad()
    def retrieve(self, input_ids: torch.Tensor, num_candidates: int = 500, exclude: Optional[torch.Tensor] = None) -> Fn.TopItems:
        """``recommend`` for up to 2048 items per row: the ``num_candidates`` (1..2048) best next items of each row as
        ``TopItems(scores, items)``, under the same rules, without forming the logits (see ``HSTU.retrieve``)."""
        Fn.check_candidates_args(num_candidates, exclude, input_ids.shape[0], input_ids.device)
        x = self.encode(input_ids)
        return Fn.head_candidates(x[:, -1, :], self.final_norm.weight, self.final_norm.bias, Fn.cast_bf16(self.item_embedding.weight),
                                  self.final_norm.eps, num_candidates, exclude)

    @torch.no_grad()
    def recommend_jagged(self, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int, top_k: int = 10,
                         exclude: Optional[torch.Tensor] = None) -> Fn.TopItems:
        """``recommend`` on a packed batch (input_ids [T], offsets [B+1], max_len as in ``forward_jagged``, positions by its batch-wide
        rule): one row of ``TopItems`` per sequence, selected from the head of its last row, offsets[b+1] - 1.  A sequence of length
        0 gets the head of a zero vector."""
        offsets = Fn.check_jagged_batch("recommend_jagged", input_ids, offsets, max_len, self.max_seq_len)
        Fn.check_topk_args(top_k, exclude, offsets.numel() - 1, input_ids.device)
        x = Fn.last_rows_jagged(self.encode_jagged(input_ids, offsets, max_len), offsets)
        return Fn.head_topk(x, self.final_norm.weight, self.final_norm.bias, Fn.cast_bf16(self.item_embedding.weight), self.final_norm.eps,
                            top_k, exclude)

    @torch.no_grad()
    def retrieve_jagged(self, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int, num_candidates: int = 500,
                        exclude: Optional[torch.Tensor] = None) -> Fn.TopItems:
        """``retrieve`` on a packed batch, under ``recommend_jagged``'s rules: up to 2048 items per sequence."""
        offsets = Fn.check_jagged_batch("retrieve_jagged", input_ids, offsets, max_len, self.max_seq_len)
        Fn.check_candidates_args(num_candidates, exclude, offsets.numel() - 1, input_ids.device)
        x = Fn.last_rows_jagged(self.encode_jagged(input_ids, offsets, max_len), offsets)
        return Fn.head_candidates(x, self.final_norm.weight, self.final_norm.bias, Fn.cast_bf16(self.item_embedding.weight),
                                  self.final_norm.eps, num_candidates, exclude)

    @torch.no_grad()
    def evaluate_batch(self, input_ids: torch.Tensor, targets: torch.Tensor, metrics: Optional[torch.Tensor] = None, *,
                       exclude: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Leave-one-out metrics of one evaluation batch, accumulated on the device into ``metrics`` ([6] fp32: Recall@{1,5,10} hit
        counts, NDCG@{1,5,10} sums): the loop of genrec/trainers/sasrec_trainer.py:39-82 without the logits or per-sample
        ``.item()`` calls.  Ranks are those of the last row of ``forward``'s logits with item 0 left out, ties to the lower id;
        ``exclude`` ([B, E] int64) and rows whose target is 0 behave as in ``HSTU.evaluate_batch``.  Divide by the number of samples
        once at the end of the evaluation."""
        Fn.check_exclude_arg(exclude, input_ids.shape[0], input_ids.device)
        x = self.encode(input_ids)
        return Fn.head_rank_metrics(x[:, -1, :], self.final_norm.weight, self.final_norm.bias, Fn.cast_bf16(self.item_embedding.weight),
                                    self.final_norm.eps, targets, metrics, exclude)

    @torch.no_grad()
    def evaluate_batch_jagged(self, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int, targets: torch.Tensor,
                              metrics: Optional[torch.Tensor] = None, *, exclude: Optional[torch.Tensor] = None, want_ranks: bool = False):
        """``evaluate_batch`` on a packed batch (input_ids [T], offsets [B+1], max_len as in ``forward_jagged``; targets [B] the
        held-out item of each sequence): each sequence is ranked from its last row, offsets[b+1] - 1, and the metrics are accumulated
        into ``metrics`` on the device.  A sequence of length 0 is not ranked (rank 0, adds nothing).  With ``want_ranks`` it returns
        (metrics, ranks [B] int32)."""
        B, T = offsets.numel() - 1, input_ids.numel()
        if tuple(targets.shape) != (B,):
            raise ValueError(f"evaluate_batch_jagged: targets must be [{B}] (one per sequence), got {tuple(targets.shape)}")
        offsets = Fn.check_jagged_batch("evaluate_batch_jagged", input_ids, offsets, max_len, self.max_seq_len)
        Fn.check_exclude_arg(exclude, B, input_ids.device)
        x = self.encode_jagged(input_ids, offsets, max_len)
        last = (offsets[1:] - 1).clamp(0, T - 1)
        ranked = torch.where(offsets[1:] > offsets[:-1], targets, torch.zeros_like(targets))
        return Fn.head_rank_metrics(x.index_select(0, last), self.final_norm.weight, self.final_norm.bias,
                                    Fn.cast_bf16(self.item_embedding.weight), self.final_norm.eps, ranked, metrics, exclude, want_ranks)
