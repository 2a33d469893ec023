"""TIGER (SURVEY.md section 8 row f4): drop-in mirror of ``genrec/models/tiger.py:88-452``.

Same constructor arguments, parameter names / shapes (a reference checkpoint loads with ``strict=True``), ``forward``,
``_encode_context``, ``_decode_step`` and ``generate`` as the reference's ``Tiger``.  Bind it with

    import genrec.models.tiger, genrec_b200.tiger
    genrec.models.tiger.Tiger = genrec_b200.tiger.Tiger

The norms are the T5 RMS norm kernels, the projections and the ReLU FFN the wgmma GEMMs of this library (ReLU and the hidden dropout
in the GEMM epilogue), attention the T5 attention core (``t5_attention._T5AttnFn``).  bf16 operands, fp32 accumulation.  The
embedding gathers, the residual adds, the dropouts on the block inputs / residual branches and the 769-class cross-entropy stay in
torch.

``generate`` projects the encoder memory's cross-attention K and V once per user (not once per beam, as the reference's expanded
memory does), runs step 0 on one row per user, and otherwise computes row for row what ``tiger_decode.generate`` on this module
computes: the same kernels on the same rows, so the beams and log-probabilities are the same bits.

``forward_jagged`` / ``generate_jagged`` / ``retrieve_jagged`` take the encoder memory packed (``data.pack_tiger``): each user's
rows without the pads of the batch's longest history, through the packed T5 attention core (INTEGRATION.md).
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import torch
import torch.nn.functional as F
from torch import nn

from . import _lib
from . import functional as Fn
from . import tiger_decode as td
from .t5_attention import T5Attention, _T5AttnFn, _bucket_map, attention_core_fwd, attention_core_fwd_jagged
from .tiger_decode import TigerGenerationOutput

__all__ = ["Tiger", "TigerOutput", "TigerGenerationOutput"]

RMS_EPS = 1e-6                      # RMSNorm / RootMeanSquareLayerNorm default (normalize.py:42, :77)
RMS_DIMS = (64, 128, 256, 384)      # widths of the RMS norm kernels
FFN_DIM = 1024                      # tiger.py:140
_SITES = {"n": 1 << 30}             # dropout sites of the FFN epilogues (the attention core numbers its own from 1)


class TigerOutput(NamedTuple):      # (tiger.py:73-78)
    logits: torch.Tensor
    loss: torch.Tensor


class _RmsNormFn(torch.autograd.Function):
    """y = w * x * rsqrt(mean(x^2) + eps) on fp32 rows."""

    @staticmethod
    def forward(ctx, x, w):
        xc = x.detach().contiguous().float()
        _, y, rstd = Fn.rmsnorm_fwd(xc, w.detach(), RMS_EPS, want_bf16=False, want_f32=True)
        ctx.save_for_backward(xc, rstd, w)
        return y

    @staticmethod
    def backward(ctx, dy):
        xc, rstd, w = ctx.saved_tensors
        dx, dw = Fn.rmsnorm_bwd(dy.contiguous().float(), xc, rstd, w.detach())
        return dx, dw


class _LinearFn(torch.autograd.Function):
    """Bias-free nn.Linear: fp32 rows -> bf16 operand -> fp32 result (in_proj / in_proj_context)."""

    @staticmethod
    def forward(ctx, x, w):
        xb = Fn.cast_rows_bf16(x.detach().contiguous().float())
        wb = Fn.cast_bf16(w)
        y, _ = Fn.linear_fwd(xb, wb, Fn.zero_bias(w.shape[0], x.device), 0)
        ctx.save_for_backward(xb, wb)
        return y.float()

    @staticmethod
    def backward(ctx, dy):
        xb, wb = ctx.saved_tensors
        dx, dw, _ = Fn.linear_bwd(Fn.cast_rows_bf16(dy.contiguous().float()), wb, xb)
        return dx, dw


class _FfnFn(torch.autograd.Function):
    """x + drop(wo(drop(relu(wi(norm2(x)))))) - the FFN half of a block (transformer.py:181-189, :323): the norm writes the bf16
    operand, ReLU and the hidden dropout run in the first GEMM's epilogue, the output dropout and the residual in the second's."""

    @staticmethod
    def forward(ctx, x, nw, wi, wo, p):
        xc = x.detach().contiguous().float()
        dev, D = xc.device, xc.shape[-1]
        xnb, _, rstd = Fn.rmsnorm_fwd(xc, nw.detach(), RMS_EPS)
        wib, wob = Fn.cast_bf16(wi), Fn.cast_bf16(wo)
        seed = Fn.dropout_seed(p)
        _SITES["n"] += 2
        site = _SITES["n"]
        y, z, h = Fn.ffn_fwd(xnb, wib, Fn.zero_bias(wi.shape[0], dev), wob, Fn.zero_bias(D, dev), xc, None, p, p, seed, None, site,
                             site + 1)
        ctx.save_for_backward(xc, rstd, xnb, z, h, wib, wob, nw)
        ctx.cfg = (p, seed, site)
        return y

    @staticmethod
    def backward(ctx, dy):
        xc, rstd, xnb, z, h, wib, wob, nw = ctx.saved_tensors
        p, seed, site = ctx.cfg
        dyc = dy.contiguous().float()
        dxn, dwi, _, dwo, _ = Fn.ffn_bwd(dyc, wib, wob, xnb, z, h, p, p, seed, None, site, site + 1)
        dx, dnw = Fn.rmsnorm_bwd(dxn, xc, rstd, nw.detach(), residual=dyc)
        return dx, dnw, dwi, dwo, None


def _head_mirrors(w: torch.Tensor):
    """bf16 copies of output_head.weight [V, D] padded with zero rows to a multiple of 8: [Vp, D] and its transpose [D, Vp]."""
    V, D = w.shape
    Vp = (V + 7) // 8 * 8
    wp = torch.zeros(Vp, D, dtype=torch.bfloat16, device=w.device)
    Fn.cast_bf16(w, wp[:V])
    return wp, wp.t().contiguous()


class _HeadFn(torch.autograd.Function):
    """output_head (tiger.py:147, :207): fp32 logits [..., V] of fp32 rows."""

    @staticmethod
    def forward(ctx, x, w):
        xb = Fn.cast_rows_bf16(x.detach().contiguous().float())
        wp, wpt = _head_mirrors(w)
        ctx.save_for_backward(xb, wp)
        ctx.V = w.shape[0]
        return Fn.matmul_f32(xb, wpt)[..., :ctx.V]

    @staticmethod
    def backward(ctx, dy):
        xb, wp = ctx.saved_tensors
        dpad = torch.zeros(*dy.shape[:-1], wp.shape[0], dtype=torch.float32, device=dy.device)
        dpad[..., :ctx.V] = dy
        dx, dw, _ = Fn.linear_bwd(Fn.cast_rows_bf16(dpad), wp, xb)
        return dx, dw[:ctx.V]


# ---- modules with the reference's parameter names (embedding.py, normalize.py, transformer.py)
class _Norm(nn.Module):
    def __init__(self, dim: int) -> None:
        super().__init__()
        self.weight = nn.Parameter(torch.ones(dim))

    def forward(self, x):
        return _RmsNormFn.apply(x, self.weight)


class _Emb(nn.Module):
    def __init__(self, n: int, dim: int, padding_idx: Optional[int] = None) -> None:
        super().__init__()
        self.emb = nn.Embedding(n, dim, padding_idx=padding_idx)


class _MHA(nn.Module):
    def __init__(self, dim: int, heads: int, dropout: float, cross: bool) -> None:
        super().__init__()
        self.attn = T5Attention(dim, heads, dropout, is_cross_attention=cross)


class _FF(nn.Module):
    def __init__(self, dim: int, hidden: int) -> None:
        super().__init__()
        self.wi = nn.Linear(dim, hidden, bias=False)
        self.wo = nn.Linear(hidden, dim, bias=False)


class _Block(nn.Module):
    def __init__(self, dim: int, heads: int, dropout: float, cross: bool) -> None:
        super().__init__()
        self.self_attn = _MHA(dim, heads, dropout, False)
        self.norm1 = _Norm(dim)
        if cross:
            self.cross_attn = _MHA(dim, heads, dropout, True)
            self.norm_cross = _Norm(dim)
        self.ff = _FF(dim, FFN_DIM)
        self.norm2 = _Norm(dim)


class _Stack(nn.Module):
    def __init__(self, dim: int, depth: int, heads: int, dropout: float, cross: bool) -> None:
        super().__init__()
        self.layers = nn.ModuleList([_Block(dim, heads, dropout, cross) for _ in range(depth)])


class _EncDec(nn.Module):
    def __init__(self, dim: int, heads: int, n_enc: int, n_dec: int, dropout: float) -> None:
        super().__init__()
        self.encoder = _Stack(dim, n_enc, heads, dropout, False)
        self.decoder = _Stack(dim, n_dec, heads, dropout, True)


class Tiger(nn.Module):
    """Mirror of genrec/models/tiger.py:88-452."""

    def __init__(self, embedding_dim: int, attn_dim: int, dropout: float, num_heads: int, n_layers: int, num_item_embeddings: int,
                 num_user_embeddings: int, sem_id_dim: int, max_pos: int = 2048) -> None:
        super().__init__()
        if attn_dim % num_heads or attn_dim // num_heads not in (32, 64):
            raise _lib.GrbError(f"genrec_b200 error -1: head_dim {attn_dim / num_heads:g} unsupported (32, 64)")
        for name, d in (("embedding_dim", embedding_dim), ("attn_dim", attn_dim)):
            if d % 8 or d not in RMS_DIMS:
                raise _lib.GrbError(f"genrec_b200 error -1: {name} {d} unsupported {RMS_DIMS}")
        self.embedding_dim, self.attn_dim, self.dropout, self.num_heads, self.n_layers = embedding_dim, attn_dim, dropout, num_heads, n_layers
        self.num_item_embeddings, self.num_user_embeddings, self.sem_id_dim, self.max_pos = (num_item_embeddings, num_user_embeddings,
                                                                                            sem_id_dim, max_pos)
        self.bos_embedding = nn.Parameter(torch.randn(embedding_dim))
        self.norm = _Norm(embedding_dim)
        self.norm_context = _Norm(embedding_dim)
        self.drop = nn.Dropout(p=dropout)
        self.sem_id_embedding = _Emb(num_item_embeddings * sem_id_dim + 1, embedding_dim, padding_idx=num_item_embeddings * sem_id_dim)
        self.user_id_embedding = _Emb(num_user_embeddings, embedding_dim)
        self.pos_embedding = nn.Embedding(max_pos, embedding_dim)                 # unused by the reference's forward, kept for checkpoints
        self.decoder_pos_embedding = nn.Embedding(sem_id_dim, embedding_dim)
        self.in_proj = nn.Linear(embedding_dim, attn_dim, bias=False)
        self.in_proj_context = nn.Linear(embedding_dim, attn_dim, bias=False)
        self.transformer = _EncDec(attn_dim, num_heads, n_layers // 2, n_layers // 2, dropout)
        self.out_proj = nn.Linear(attn_dim, embedding_dim, bias=False)
        self.vocab_size = num_item_embeddings * sem_id_dim + 1
        self.output_head = nn.Linear(attn_dim, self.vocab_size, bias=False)

    # ---- pieces
    def _p(self) -> float:
        return self.dropout if self.training else 0.0

    def _sem_emb(self, ids, types):
        return self.sem_id_embedding.emb(types * self.num_item_embeddings + ids)          # embedding.py:42-43

    def _context_input(self, user_input_ids, item_input_ids, token_type_ids, seq_mask):
        """-> (encoder input [B, 1+N, attn_dim] fp32, key padding [B, 1+N] bool)"""
        user_emb = self.user_id_embedding.emb(user_input_ids % self.num_user_embeddings)   # embedding.py:73-74
        x = torch.cat([user_emb, self._sem_emb(item_input_ids, token_type_ids)], dim=1)
        pad = torch.cat([torch.zeros(seq_mask.size(0), 1, dtype=torch.bool, device=seq_mask.device), seq_mask == 0], dim=1)
        x = _LinearFn.apply(F.dropout(self.norm_context(x), self._p(), self.training), self.in_proj_context.weight)
        return x, pad

    def _decoder_input(self, B: int, tgt_ids, tgt_type):
        bos = self.bos_embedding.view(1, 1, -1).expand(B, 1, -1)
        x = bos if tgt_ids is None else torch.cat([bos, self._sem_emb(tgt_ids, tgt_type)], dim=1)
        return _LinearFn.apply(F.dropout(self.norm(x), self._p(), self.training), self.in_proj.weight)

    def _self_attn(self, blk, x, pad, causal, jagged=None):
        """jagged = (offsets, max_len): x [T, D] holds the packed sequences (no key padding)"""
        a = blk.self_attn.attn
        L = x.shape[1] if jagged is None else jagged[1]
        bucket = _bucket_map(L, L, a.num_relative_buckets, a.max_distance, x.device)
        kp = pad.to(torch.uint8).contiguous() if pad is not None else None
        out = _T5AttnFn.apply(blk.norm1(x), None, None, kp, causal, a.n_heads, self._p(), bucket, a.q.weight, a.kv.weight, None,
                              a.o.weight, a.rel_bias.weight, True, *(jagged or ()))
        return x + F.dropout(out, self._p(), self.training)

    def _ffn(self, blk, x):
        return _FfnFn.apply(x, blk.norm2.weight, blk.ff.wi.weight, blk.ff.wo.weight, self._p())

    def _encoder(self, x, pad, jagged=None):
        for blk in self.transformer.encoder.layers:                                      # transformer.py:363-365, :303-324
            x = self._ffn(blk, self._self_attn(blk, x, pad, False, jagged))
        return x

    def _cross(self, blk, x, memory, memory_pad, jagged=None):
        """jagged = (offsets, max_len): memory [T, D] holds the packed sequences, memory_pad is None"""
        a = blk.cross_attn.attn
        kp = memory_pad.to(torch.uint8).contiguous() if memory_pad is not None else None
        out = _T5AttnFn.apply(blk.norm_cross(x), memory, memory, kp, False, a.n_heads, self._p(), None, a.q.weight, a.k.weight, a.v.weight,
                              a.o.weight, None, False, *(jagged or ()))
        return x + F.dropout(out, self._p(), self.training)

    def _decoder(self, x, cross):
        for i, blk in enumerate(self.transformer.decoder.layers):                        # transformer.py:406-414, :303-324
            x = self._self_attn(blk, x, None, True)
            x = cross(i, blk, x)
            x = self._ffn(blk, x)
        return x

    # ---- packed (jagged) encoder memory
    def _check_jagged(self, what, user_input_ids, item_input_ids, token_type_ids, mem_offsets, max_len):
        """ValueError before anything runs -> (user ids [B], offsets on the device)"""
        if not isinstance(token_type_ids, torch.Tensor) or token_type_ids.shape != item_input_ids.shape:
            raise ValueError(f"{what}: token_type_ids must be [T] like item_input_ids, got "
                             f"{tuple(token_type_ids.shape) if isinstance(token_type_ids, torch.Tensor) else token_type_ids!r}")
        users = user_input_ids.reshape(-1)
        if isinstance(mem_offsets, torch.Tensor) and mem_offsets.dim() == 1:
            if users.numel() != mem_offsets.numel() - 1:
                raise ValueError(f"{what}: {users.numel()} user ids for {mem_offsets.numel() - 1} sequences")
            if not mem_offsets.is_cuda and bool(((mem_offsets[1:] - mem_offsets[:-1]) == 0).any()):
                raise ValueError(f"{what}: every sequence starts with its user row (length >= 1)")
        return users, Fn.check_jagged_batch(what, item_input_ids, mem_offsets, max_len, self.max_pos)

    def _encode_context_jagged(self, users, item_input_ids, token_type_ids, offsets, max_len):
        """-> encoder memory [T, attn_dim] fp32: row offsets[b] is user b's token (its item_input_ids / token_type_ids are ignored),
        the rows behind it its item tokens - Tiger.forward's [user, items] without the pads."""
        x = self._sem_emb(item_input_ids, token_type_ids)
        user_emb = self.user_id_embedding.emb(users % self.num_user_embeddings)
        x = x.index_put((offsets[:-1].clamp(max=x.size(0) - 1),), user_emb)
        x = _LinearFn.apply(F.dropout(self.norm_context(x), self._p(), self.training), self.in_proj_context.weight)
        return self._encoder(x, None, (offsets, max_len))

    def forward_jagged(self, user_input_ids, item_input_ids, token_type_ids, mem_offsets, max_len: int, target_input_ids,
                       target_token_type_ids) -> TigerOutput:
        """``forward`` on a packed encoder memory (``data.pack_tiger``): user b's memory is rows mem_offsets[b] .. mem_offsets[b+1]-1
        of item_input_ids / token_type_ids [T] (its user row first), at most max_len rows; user_input_ids [B] (or [B, 1]); the
        decoder input stays [B, S].  Returns logits [B, S+1, V] and the reference's loss (sum over positions, mean over users): on the
        same users the values of ``forward`` on pad_collate's batch, without computing the pads.  Rows past mem_offsets[B] are idle.
        Dropout draws its encoder self-attention masks by token row, so under dropout a packed batch draws other masks than the
        padded one.  Refusals are ValueError before anything runs; device offsets are not read on the host."""
        users, offsets = self._check_jagged("Tiger.forward_jagged", user_input_ids, item_input_ids, token_type_ids, mem_offsets, max_len)
        B = users.numel()
        memory = self._encode_context_jagged(users, item_input_ids, token_type_ids, offsets, max_len)
        tgt = self._decoder_input(B, target_input_ids, target_token_type_ids)
        out = self._decoder(tgt, lambda i, blk, x: self._cross(blk, x, memory, None, (offsets, max_len)))
        return self._output(B, out, target_input_ids, target_token_type_ids)

    @torch.no_grad()
    def generate_jagged(self, user_input_ids, item_input_ids, token_type_ids, mem_offsets, max_len: int, temperature: float = 0.2,
                        n_top_k_candidates: int = 10, valid_item_ids=None, use_trie: bool = True,
                        generator: Optional[torch.Generator] = None) -> TigerGenerationOutput:
        """``generate`` on a packed encoder memory (the layout of ``forward_jagged``): the same beams and log-probabilities as
        ``generate`` on the padded batch of the same users.  No host synchronisation once the trie is built, so with device offsets a
        warmed-up call can be captured in a CUDA graph and replayed with other ids and offsets of the same T and max_len."""
        users, offsets = self._check_jagged("Tiger.generate_jagged", user_input_ids, item_input_ids, token_type_ids, mem_offsets, max_len)
        out, _, _ = self._generate(users, item_input_ids, token_type_ids, None, temperature, n_top_k_candidates, valid_item_ids, use_trie,
                                   generator, jagged=(offsets, max_len))
        return out

    @torch.no_grad()
    def retrieve_jagged(self, user_input_ids, item_input_ids, token_type_ids, mem_offsets, max_len: int, num_candidates: int = 500,
                        valid_item_ids=None, temperature: float = 0.2, generator: Optional[torch.Generator] = None):
        """``retrieve`` on a packed encoder memory: (items [B, K], sem_ids [B, K, sem_id_dim], log_probas [B, K])."""
        users, offsets = self._check_jagged("Tiger.retrieve_jagged", user_input_ids, item_input_ids, token_type_ids, mem_offsets, max_len)
        out, nodes, trie = self._generate(users, item_input_ids, token_type_ids, None, temperature, num_candidates, valid_item_ids, True,
                                          generator, want_nodes=True, jagged=(offsets, max_len))
        return trie.rows(nodes), out.sem_ids, out.log_probas

    def _output(self, B, out, target_input_ids, target_token_type_ids) -> TigerOutput:
        logits = _HeadFn.apply(out, self.output_head.weight)
        loss = None
        if target_input_ids is not None and target_input_ids.shape[1] == self.sem_id_dim:   # tiger.py:232-242
            target_vocab_ids = target_token_type_ids * self.num_item_embeddings + target_input_ids
            loss_logits = logits[:, :-1, :]
            loss = F.cross_entropy(loss_logits.reshape(-1, loss_logits.size(-1)), target_vocab_ids.reshape(-1),
                                   reduction="none").reshape(B, -1).sum(dim=1).mean()
        return TigerOutput(logits=logits, loss=loss)

    # ---- the reference's interface
    def forward(self, user_input_ids, item_input_ids, token_type_ids, target_input_ids, target_token_type_ids, seq_mask) -> TigerOutput:
        if seq_mask is None:
            seq_mask = torch.ones_like(item_input_ids, dtype=torch.long, device=item_input_ids.device)
        B = item_input_ids.size(0)
        src, pad = self._context_input(user_input_ids, item_input_ids, token_type_ids, seq_mask)
        tgt = self._decoder_input(B, target_input_ids, target_token_type_ids)
        memory = self._encoder(src, pad)
        out = self._decoder(tgt, lambda i, blk, x: self._cross(blk, x, memory, pad))
        return self._output(B, out, target_input_ids, target_token_type_ids)

    def _encode_context(self, user_input_ids, item_input_ids, token_type_ids, seq_mask=None):
        if seq_mask is None:
            seq_mask = torch.ones_like(item_input_ids, dtype=torch.long, device=item_input_ids.device)
        src, pad = self._context_input(user_input_ids, item_input_ids, token_type_ids, seq_mask)
        return self._encoder(src, pad), pad

    def _decode_step(self, memory, memory_mask, tgt_ids, tgt_type):
        x = self._decoder_input(memory.size(0), tgt_ids, tgt_type)
        out = self._decoder(x, lambda i, blk, h: self._cross(blk, h, memory, memory_mask))
        return _HeadFn.apply(out[:, -1], self.output_head.weight)

    @torch.no_grad()
    def generate(self, user_input_ids, item_input_ids, token_type_ids, seq_mask=None, temperature: float = 0.2, n_top_k_candidates: int = 10,
                 valid_item_ids=None, use_trie: bool = True, generator: Optional[torch.Generator] = None) -> TigerGenerationOutput:
        """Trie-constrained beam search (tiger.py:312-452) with the memory's cross-attention K / V projected once per user.  No host
        synchronisation once the trie is built (first call), so a warmed-up call can be captured in a CUDA graph.  1 <= K <= 1024
        beams per user with K * min(6 K, num_item_embeddings) <= 262,144 (ValueError before anything runs otherwise)."""
        out, _, _ = self._generate(user_input_ids, item_input_ids, token_type_ids, seq_mask, temperature, n_top_k_candidates, valid_item_ids,
                                   use_trie, generator)
        return out

    @torch.no_grad()
    def retrieve(self, user_input_ids, item_input_ids, token_type_ids, seq_mask=None, num_candidates: int = 500, valid_item_ids=None,
                 temperature: float = 0.2, generator: Optional[torch.Generator] = None):
        """Candidates for a ranker: ``generate`` with the trie, plus the catalog row of each beam's item.  Returns (items [B, K] int64,
        sem_ids [B, K, sem_id_dim], log_probas [B, K]); items are rows of ``valid_item_ids`` (the smallest row holding the beam's
        tuple), -1 for filler beams and for beams whose sequence left the trie.  The beams are ``generate``'s under the same generator
        state."""
        out, nodes, trie = self._generate(user_input_ids, item_input_ids, token_type_ids, seq_mask, temperature, num_candidates,
                                          valid_item_ids, True, generator, want_nodes=True)
        return trie.rows(nodes), out.sem_ids, out.log_probas

    def _generate(self, user_input_ids, item_input_ids, token_type_ids, seq_mask, temperature, K, valid_item_ids, use_trie, generator,
                  want_nodes=False, jagged=None):
        """-> (beams, final trie nodes if want_nodes else None, trie); the arguments are checked before anything runs.  jagged =
        (offsets, max_len): the memory is packed (``generate_jagged``)."""
        td.check_width(K, td.candidates_per_beam(K, self.num_item_embeddings))
        B = user_input_ids.size(0)
        dev = user_input_ids.device
        trie = None
        if use_trie:
            trie = getattr(self, "_grb_trie", None)
            if trie is None:
                if valid_item_ids is None:
                    raise ValueError("the trie is built from valid_item_ids on the first call")
                trie = td.TrieCSR.build(valid_item_ids).to(dev)
                self._grb_trie = trie
        if jagged is None:
            memory, memory_pad = self._encode_context(user_input_ids, item_input_ids, token_type_ids, seq_mask)
            kp = memory_pad.to(torch.uint8).contiguous()
        else:
            memory = self._encode_context_jagged(user_input_ids, item_input_ids, token_type_ids, *jagged)
        xm = Fn.cast_rows_bf16(memory.contiguous())
        D = self.attn_dim
        mem_kv = []                                                  # per decoder block: K, V [B, 1+N, D] (packed: [T, D]) bf16
        for blk in self.transformer.decoder.layers:
            a = blk.cross_attn.attn
            Km, _ = Fn.linear_fwd(xm, Fn.cast_bf16(a.k.weight), Fn.zero_bias(D, dev), 0)
            Vm, _ = Fn.linear_fwd(xm, Fn.cast_bf16(a.v.weight), Fn.zero_bias(D, dev), 0)
            mem_kv.append((Km, Vm))
        wcache = [(Fn.cast_bf16(b.cross_attn.attn.q.weight), Fn.cast_bf16(b.cross_attn.attn.o.weight)) for b in self.transformer.decoder.layers]
        H = self.num_heads
        scale = 1.0 / math.sqrt(D // H)

        def cross(i, blk, x):
            # the queries of a user's beams against that user's memory: [B*R, S, D] viewed as [B, R*S, D]
            R, S = x.size(0) // B, x.size(1)
            wq, wo = wcache[i]
            Q, _ = Fn.linear_fwd(Fn.cast_rows_bf16(blk.norm_cross(x).contiguous()), wq, Fn.zero_bias(D, dev), 0)
            if jagged is None:
                A, _ = attention_core_fwd(Q.view(B, R * S, D), mem_kv[i][0], mem_kv[i][1], H, None, None, kp, False, scale)
            else:
                A, _ = attention_core_fwd_jagged(Q.view(B, R * S, D), mem_kv[i][0], mem_kv[i][1], H, None, None, *jagged, False, scale)
            out, _ = Fn.linear_fwd(A.view(B * R, S, D), wo, Fn.zero_bias(D, dev), 0)
            return x + out.float()

        wp, wpt = _head_mirrors(self.output_head.weight)
        V = self.vocab_size

        def decode_step(tgt):
            if tgt.size(1) == 0:                                     # every beam is [bos]: one row per user, logits broadcast
                x = self._decoder_input(B, None, None)
                rows = B
            else:
                types = torch.arange(tgt.size(1), device=dev).unsqueeze(0).expand(tgt.size(0), -1)
                x = self._decoder_input(tgt.size(0), tgt, types)
                rows = tgt.size(0)
            out = self._decoder(x, cross)
            logits = Fn.matmul_f32(Fn.cast_rows_bf16(out[:, -1].contiguous()), wpt)[..., :V]
            return logits if rows == B * K else logits.unsqueeze(1).expand(B, K, V).reshape(B * K, V)

        run = (B, K, self.sem_id_dim, self.num_item_embeddings, dev, temperature, trie, generator)
        if want_nodes:
            out, nodes = td.beam_search(decode_step, *run, return_nodes=True)
            return out, nodes, trie
        return td.beam_search(decode_step, *run), None, trie
