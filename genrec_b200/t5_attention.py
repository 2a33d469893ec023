"""T5-style attention for TIGER (SURVEY.md section 8 row f4): drop-in mirror of ``genrec/modules/transformer.py:44-159``.

Same constructor arguments, parameter names / shapes (``q``, ``kv`` | ``k`` + ``v``, ``o``, ``rel_bias``) and ``forward`` signature as
the reference's ``T5Attention``; the q / k / v / o projections are the wgmma GEMMs of this library, the score / softmax / value core
is ``csrc/attn_t5.cuh`` (forward and backward), glued by one autograd function.  bf16 operands, fp32 accumulation, like the other
modules of this package.  Supported masks: ``key_padding_mask`` [B, Lk] bool and ``attn_mask`` = None or the causal mask of
``nn.Transformer.generate_square_subsequent_mask`` (what genrec/models/tiger.py:203-206,306-309 passes); anything else raises.
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
from torch import nn

from . import functional as Fn
from . import _lib
from ._lib import call, ptr, require_cuda, ensure_device, workspace

_CALLS = {"n": 0}
_BUCKETS, _CAUSAL = {}, {}


def relative_position_buckets(q_len: int, k_len: int, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """Bucket of every delta = j - i, i in [0, q_len), j in [0, k_len): int32 [q_len + k_len - 1], index delta + q_len - 1.
    Bidirectional T5 bucketing exactly as transformer.py:13-41 evaluates it (same fp32 log expression, same truncation)."""
    delta = torch.arange(-(q_len - 1), k_len, dtype=torch.long)          # memory position - context position
    n = -delta
    half = num_buckets // 2
    side = (n < 0).long() * half
    n = n.abs()
    exact = half // 2
    large = exact + (torch.log(n.float() / exact + 1e-6) / math.log(max_distance / exact) * (half - exact)).long().clamp(max=half - exact - 1)
    return (torch.where(n < exact, n, large) + side).to(torch.int32)


def _bucket_map(q_len, k_len, nb, maxd, device) -> torch.Tensor:
    key = (q_len, k_len, nb, maxd, str(device))
    if key not in _BUCKETS:
        _BUCKETS[key] = relative_position_buckets(q_len, k_len, nb, maxd).to(device)
    return _BUCKETS[key]


def _is_causal(attn_mask: Optional[torch.Tensor], q_len: int, k_len: int) -> bool:
    if attn_mask is None:
        return False
    m = attn_mask
    while m.dim() > 2 and m.size(0) == 1:
        m = m[0]
    key = (m.data_ptr(), tuple(m.shape), m._version)
    if key not in _CAUSAL:
        ok = m.dim() == 2 and tuple(m.shape) == (q_len, k_len) and q_len == k_len and m.dtype.is_floating_point
        if ok:
            ref = torch.triu(torch.full((q_len, k_len), float("-inf"), device=m.device, dtype=m.dtype), diagonal=1)
            ok = bool(torch.equal(m, ref))
        _CAUSAL.clear()
        _CAUSAL[key] = ok
    if not _CAUSAL[key]:
        raise NotImplementedError("genrec_b200.T5Attention: attn_mask must be None or the causal (square subsequent) float mask")
    return True


def attention_core_fwd(Q, K, V, H, bias, bucket, key_pad, causal, scale, p=0.0, seed=0, site=0):
    """Q [B, Lq, *] / K, V [B, Lk, *] bf16 (last-dim views allowed) -> (out bf16 [B, Lq, D], softmax statistics fp32 [B, H, Lq, 2])."""
    B, Lq, D = Q.shape
    Lk = K.shape[1]
    out = torch.empty(B, Lq, D, dtype=torch.bfloat16, device=Q.device)
    lse = torch.empty(B, H, Lq, 2, dtype=torch.float32, device=Q.device)     # {row max, sum of exp(s - max)}
    nb = bias.shape[1] if bias is not None else 0
    call(Q.device, "grb_t5_attention_forward", ptr(Q), ptr(K), ptr(V), B, Lq, Lk, H, D // H, Q.stride(1), K.stride(1), V.stride(1),
         ptr(bias), ptr(bucket), nb, ptr(key_pad), 1 if causal else 0, float(scale), float(p), int(seed), None, int(site) & 0xFFFFFFFF,
         ptr(out), D, ptr(lse))
    return out, lse


def attention_core_bwd(Q, K, V, H, bias, bucket, key_pad, causal, scale, out, lse, dout, p=0.0, seed=0, site=0):
    B, Lq, D = Q.shape
    Lk = K.shape[1]
    dq = torch.empty(B, Lq, D, dtype=torch.bfloat16, device=Q.device)
    dk = torch.empty(B, Lk, D, dtype=torch.float32, device=Q.device)
    dv = torch.empty(B, Lk, D, dtype=torch.float32, device=Q.device)
    dbias = torch.zeros_like(bias) if bias is not None else None
    nb = bias.shape[1] if bias is not None else 0
    ws = workspace(Q.device, "grb_t5_attention_backward_workspace_bytes", B, Lq, Lk, H, D // H, nb, allow_empty=True)
    call(Q.device, "grb_t5_attention_backward", ptr(Q), ptr(K), ptr(V), B, Lq, Lk, H, D // H, Q.stride(1), K.stride(1), V.stride(1),
         ptr(bias), ptr(bucket), nb, ptr(key_pad), 1 if causal else 0, float(scale), float(p), int(seed), None, int(site) & 0xFFFFFFFF,
         ptr(out), D, ptr(lse), ptr(dout), D, ptr(dq), D, ptr(dk), ptr(dv), ptr(dbias), ptr(ws) if ws.numel() else None)
    return dq, dk, dv, dbias


def _jagged_shape(Q, K, max_len):
    """(B, T, Lq) of a packed call: Q [T, D] (self-attention, Lq = 0: the queries are the packed rows) or [B, Lq, D] (cross-attention,
    the keys K [T, D] are packed)."""
    return (None, Q.shape[0], 0) if Q.dim() == 2 else (Q.shape[0], K.shape[0], Q.shape[1])


def attention_core_fwd_jagged(Q, K, V, H, bias, bucket, offsets, max_len, causal, scale, p=0.0, seed=0, site=0):
    """``attention_core_fwd`` on a packed batch (``grb_t5_attention_forward_jagged``): sequence b is rows offsets[b] .. offsets[b+1]-1
    of the packed K / V [T, *] (and of Q [T, *] in self-attention; Q [B, Lq, *] stays dense in cross-attention).  bucket is
    ``relative_position_buckets(Lq or max_len, max_len)``.  -> (out like Q, softmax statistics [H, T, 2] or [B, H, Lq, 2])."""
    _, T, Lq = _jagged_shape(Q, K, max_len)
    B = offsets.numel() - 1
    D = Q.shape[-1]
    out = torch.empty(*Q.shape[:-1], D, dtype=torch.bfloat16, device=Q.device)
    lse = torch.empty(*((H, T) if Lq == 0 else (B, H, Lq)), 2, dtype=torch.float32, device=Q.device)
    nb = bias.shape[1] if bias is not None else 0
    call(Q.device, "grb_t5_attention_forward_jagged",
         ptr(Q), ptr(K), ptr(V), ptr(offsets), B, T, int(max_len), Lq, H, D // H, Q.stride(-2), K.stride(-2), V.stride(-2), ptr(bias),
         ptr(bucket), bucket.numel() if bucket is not None else 0, nb, 1 if causal else 0, float(scale), float(p), int(seed), None,
         int(site) & 0xFFFFFFFF, ptr(out), D, ptr(lse))
    return out, lse


def attention_core_bwd_jagged(Q, K, V, H, bias, bucket, offsets, max_len, causal, scale, out, lse, dout, p=0.0, seed=0, site=0):
    """``attention_core_bwd`` on a packed batch: -> (dq like Q bf16, dk, dv [T, D] fp32, dbias)."""
    _, T, Lq = _jagged_shape(Q, K, max_len)
    B = offsets.numel() - 1
    D = Q.shape[-1]
    dq = torch.empty(*Q.shape[:-1], D, dtype=torch.bfloat16, device=Q.device)
    dk = torch.empty(T, D, dtype=torch.float32, device=Q.device)
    dv = torch.empty(T, D, dtype=torch.float32, device=Q.device)
    dbias = torch.zeros_like(bias) if bias is not None else None
    nb = bias.shape[1] if bias is not None else 0
    ws = workspace(Q.device, "grb_t5_attention_backward_workspace_bytes_jagged", B, T, int(max_len), Lq, H, D // H, nb, allow_empty=True)
    call(Q.device, "grb_t5_attention_backward_jagged",
         ptr(Q), ptr(K), ptr(V), ptr(offsets), B, T, int(max_len), Lq, H, D // H, Q.stride(-2), K.stride(-2), V.stride(-2), ptr(bias),
         ptr(bucket), bucket.numel() if bucket is not None else 0, nb, 1 if causal else 0, float(scale), float(p), int(seed), None,
         int(site) & 0xFFFFFFFF, ptr(out), D, ptr(lse), ptr(dout), D, ptr(dq), D, ptr(dk), ptr(dv), ptr(dbias),
         ptr(ws) if ws.numel() else None)
    return dq, dk, dv, dbias


class _T5AttnFn(torch.autograd.Function):
    """T5Attention.forward as a unit: projections, attention core, output projection.  With ``offsets`` [B+1] (device) and
    ``max_len`` the batch is packed: the query rows [T, D] in self-attention, the key / value rows [T, D] in cross-attention."""

    @staticmethod
    def forward(ctx, query, key, value, key_pad, causal, H, p, bucket, wq, wk, wv, wo, rel_w, fused_kv, offsets=None, max_len=0):
        require_cuda(query)
        ensure_device(query.device)
        dev = query.device
        D = query.shape[-1]
        xq = Fn.cast_rows_bf16(query.detach().contiguous().float())
        wqb, wob = Fn.cast_bf16(wq), Fn.cast_bf16(wo)
        Q, _ = Fn.linear_fwd(xq, wqb, Fn.zero_bias(D, dev), 0)
        if fused_kv:                                   # self-attention: one [2D, D] projection of the query stream (transformer.py:121-123)
            wkb = Fn.cast_bf16(wk)                     # wk holds the kv weight
            KV, _ = Fn.linear_fwd(xq, wkb, Fn.zero_bias(2 * D, dev), 0)
            K, V = KV[..., :D], KV[..., D:]
            xk = xv = xq
            wvb = None
        else:                                          # cross-attention (transformer.py:117-119)
            xk = Fn.cast_rows_bf16(key.detach().contiguous().float())
            xv = xk if value is key else Fn.cast_rows_bf16(value.detach().contiguous().float())
            wkb, wvb = Fn.cast_bf16(wk), Fn.cast_bf16(wv)
            K, _ = Fn.linear_fwd(xk, wkb, Fn.zero_bias(D, dev), 0)
            V, _ = Fn.linear_fwd(xv, wvb, Fn.zero_bias(D, dev), 0)
        bias = rel_w.detach().float().view(H, -1).contiguous() if rel_w is not None else None
        seed = Fn.dropout_seed(p)
        _CALLS["n"] += 1
        site = _CALLS["n"]
        scale = 1.0 / math.sqrt(D // H)
        if offsets is None:
            A, lse = attention_core_fwd(Q, K, V, H, bias, bucket, key_pad, causal, scale, p, seed, site)
        else:
            A, lse = attention_core_fwd_jagged(Q, K, V, H, bias, bucket, offsets, max_len, causal, scale, p, seed, site)
        out, _ = Fn.linear_fwd(A, wob, Fn.zero_bias(D, dev), 0)
        ctx.save_for_backward(xq, xk, xv, Q, K, V, A, lse, wqb, wkb, wvb if wvb is not None else wqb, wob, bias if bias is not None else lse,
                              bucket if bucket is not None else lse, key_pad if key_pad is not None else lse,
                              offsets if offsets is not None else lse)
        ctx.cfg = (H, p, seed, site, scale, causal, fused_kv, bias is not None, key_pad is not None, value is key)
        ctx.jagged = (offsets is not None, max_len)
        return out.float()

    @staticmethod
    def backward(ctx, dout):
        xq, xk, xv, Q, K, V, A, lse, wqb, wkb, wvb, wob, bias, bucket, key_pad, offsets = ctx.saved_tensors
        H, p, seed, site, scale, causal, fused_kv, has_bias, has_pad, same_kv = ctx.cfg
        jagged, max_len = ctx.jagged
        bias = bias if has_bias else None
        bucket = bucket if has_bias else None
        key_pad = key_pad if has_pad else None
        dyb = Fn.cast_rows_bf16(dout.contiguous().float())
        dA, dwo, _ = Fn.linear_bwd(dyb, wob, A)
        if jagged:
            dQ, dK32, dV32, dbias = attention_core_bwd_jagged(Q, K, V, H, bias, bucket, offsets, max_len, causal, scale, A, lse,
                                                              Fn.cast_rows_bf16(dA), p, seed, site)
        else:
            dQ, dK32, dV32, dbias = attention_core_bwd(Q, K, V, H, bias, bucket, key_pad, causal, scale, A, lse, Fn.cast_rows_bf16(dA), p,
                                                       seed, site)
        if fused_kv:
            dKV = Fn.cast_rows_bf16(torch.cat([dK32, dV32], dim=-1))
            dx_kv, dwkv, _ = Fn.linear_bwd(dKV, wkb, xq)
            dquery, dwq, _ = Fn.linear_bwd(dQ, wqb, xq, dx_residual=dx_kv)
            dkey = dvalue = None
            dwk, dwv = dwkv, None
        else:
            dquery, dwq, _ = Fn.linear_bwd(dQ, wqb, xq)
            dkey, dwk, _ = Fn.linear_bwd(Fn.cast_rows_bf16(dK32), wkb, xk)
            dvalue, dwv, _ = Fn.linear_bwd(Fn.cast_rows_bf16(dV32), wvb, xv)
        drel = dbias.reshape(-1, 1) if has_bias else None
        return dquery, dkey, dvalue, None, None, None, None, None, dwq, dwk, dwv, dwo, drel, None, None, None


class T5Attention(nn.Module):
    """Mirror of genrec/modules/transformer.py:44-159."""

    def __init__(self, d_model: int, n_heads: int, dropout: float = 0.0, is_cross_attention: bool = False, has_relative_bias: bool = True,
                 num_relative_buckets: int = 32, max_distance: int = 128) -> None:
        super().__init__()
        assert d_model % n_heads == 0
        self.d_model, self.n_heads, self.head_dim = d_model, n_heads, d_model // n_heads
        self.scale = 1.0 / math.sqrt(self.head_dim)
        self.is_cross_attention, self.has_relative_bias = is_cross_attention, has_relative_bias
        self.q = nn.Linear(d_model, d_model, bias=False)
        if is_cross_attention:
            self.k = nn.Linear(d_model, d_model, bias=False)
            self.v = nn.Linear(d_model, d_model, bias=False)
        else:
            self.kv = nn.Linear(d_model, 2 * d_model, bias=False)
        self.o = nn.Linear(d_model, d_model, bias=False)
        self.dropout = nn.Dropout(dropout)
        if has_relative_bias and not is_cross_attention:
            self.rel_bias = nn.Embedding(n_heads * num_relative_buckets, 1)
            self.num_relative_buckets, self.max_distance = num_relative_buckets, max_distance
        else:
            self.rel_bias = None

    def _get_rel_bias(self, q_len: int, k_len: int, device) -> torch.Tensor:
        """[1, H, q_len, k_len] bias tensor (transformer.py:84-104) - only materialised for callers that ask for it."""
        b = _bucket_map(q_len, k_len, self.num_relative_buckets, self.max_distance, device).long()
        i = torch.arange(q_len, device=device)[:, None]
        j = torch.arange(k_len, device=device)[None, :]
        idx = b[(j - i) + q_len - 1]
        table = self.rel_bias.weight.view(self.n_heads, self.num_relative_buckets)
        return table[:, idx].unsqueeze(0)

    def forward(self, query: torch.Tensor, key: Optional[torch.Tensor] = None, value: Optional[torch.Tensor] = None,
                attn_mask: Optional[torch.Tensor] = None, key_padding_mask: Optional[torch.Tensor] = None,
                position_bias: Optional[torch.Tensor] = None, need_weights: bool = False) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        if position_bias is not None:
            raise NotImplementedError("genrec_b200.T5Attention: an externally supplied position_bias is not supported")
        if self.head_dim not in (32, 64) or self.d_model % 8:
            raise _lib.GrbError(f"genrec_b200 error -1: head_dim {self.head_dim} unsupported (32, 64)")
        require_cuda(query)
        B, Lq, _ = query.shape
        if self.is_cross_attention:
            Lk = key.shape[1]
            fused, wk, wv = False, self.k.weight, self.v.weight
        else:
            key = value = None
            Lk = Lq
            fused, wk, wv = True, self.kv.weight, None
        causal = _is_causal(attn_mask, Lq, Lk)
        pad = key_padding_mask.to(torch.uint8).contiguous() if key_padding_mask is not None else None
        bucket = _bucket_map(Lq, Lk, self.num_relative_buckets, self.max_distance, query.device) if self.rel_bias is not None else None
        out = _T5AttnFn.apply(query, key, value, pad, causal, self.n_heads, self.dropout.p if self.training else 0.0, bucket, self.q.weight, wk,
                              wv, self.o.weight, self.rel_bias.weight if self.rel_bias is not None else None, fused)
        # the reference also hands back the bias tensor it added (transformer.py:159); callers in the reference ignore it
        return out, (self._get_rel_bias(Lq, Lk, query.device).detach() if self.rel_bias is not None else None)
