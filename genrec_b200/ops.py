"""``torch.ops.genrec_b200.*`` - the hot path as dispatcher-registered PyTorch custom ops (north_star: "exposed as torch custom ops";
SURVEY.md section 8b).

Each op is a thin, tensor-only front of one C-ABI entry point (include/genrec_b200.h): tensors and scalars in, fresh tensors out, no
Python objects in the signature.  Registered with ``torch.library.custom_op`` so that they
  * appear under ``torch.ops.genrec_b200`` with a schema,
  * carry FakeTensor / meta implementations (``torch.compile``, ``make_fx`` and shape propagation trace through them without a GPU),
  * are wired into autograd with ``register_autograd`` (backward = another registered op, so double tracing works too).
They run the CUDA kernels only - a CPU tensor raises, exactly like the module API.  The nn.Module mirrors (hstu.py, sasrec.py,
rqvae.py) call the same C entry points; the grad-sink fast path of FlatAdam mutates a flat gradient buffer and therefore stays an
``autograd.Function`` (functional.py)."""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Tuple

import torch
from torch import Tensor
from torch.library import custom_op

from . import _lib
from . import functional as Fn
from ._lib import HstuDims, HstuLayerGrads, HstuLayerParams, HstuSeq, check, ptr, require_cuda, stream_ptr

NS = "genrec_b200"


def _seq(pad: Tensor, ts: Optional[Tensor], rel32: Optional[Tensor], wide: Optional[Tensor], thr: Tensor, pos_bucket0: int,
         ntime: int) -> HstuSeq:
    """Sequence metadata with the [B, L, ld] bias-index matrix the attention kernels read (uniform position buckets: one
    effective bucket).  The struct holds a reference to the index tensor, which lives as long as the struct."""
    B, L = pad.shape
    ld = (L + 7) // 8 * 8
    index = torch.empty(B, L, ld, dtype=torch.int16, device=pad.device)
    zero_pb = torch.zeros(L, dtype=torch.uint8, device=pad.device)
    pad = pad.contiguous()
    Fn._defer_for_call(False)   # built on the caller's stream: the kernels that read it and the tensor's lifetime follow that stream
    with torch.cuda.device(pad.device):
        check(_lib.load().grb_hstu_bias_index(ptr(ts), ptr(pad), ptr(thr), ptr(zero_pb), B, L, 1, ntime if ts is not None else 0, ptr(index), ld,
                                              stream_ptr(pad.device)))
    seq = HstuSeq(ptr(index), ld, 1 if ts is not None else 0, 1, int(pos_bucket0), ptr(ts), ptr(pad), ptr(rel32), ptr(wide), ptr(thr))
    seq.index = index
    return seq


# ------------------------------------------------------------------------------------------------ sequence preparation
@custom_op(f"{NS}::hstu_seq_prepare", mutates_args=())
def hstu_seq_prepare(timestamps: Tensor, pad: Tensor) -> Tuple[Tensor, Tensor]:
    """timestamps [B, L] int64, pad [B, L] uint8 -> rel32 [B, L] int32, wide [B] uint8 (grb_hstu_seq_prepare)."""
    require_cuda(timestamps, pad)
    B, L = timestamps.shape
    rel = torch.empty(B, L, dtype=torch.int32, device=pad.device)
    wide = torch.empty(B, dtype=torch.uint8, device=pad.device)
    with torch.cuda.device(pad.device):
        check(_lib.load().grb_hstu_seq_prepare(ptr(timestamps.contiguous()), ptr(pad.contiguous()), B, L, ptr(rel), ptr(wide), stream_ptr(pad.device)))
    return rel, wide


@hstu_seq_prepare.register_fake
def _(timestamps, pad):
    B, L = timestamps.shape
    return timestamps.new_empty((B, L), dtype=torch.int32), timestamps.new_empty((B,), dtype=torch.uint8)


# ------------------------------------------------------------------------------------------------ attention core
@custom_op(f"{NS}::hstu_attention", mutates_args=())
def hstu_attention(P: Tensor, pad: Tensor, timestamps: Optional[Tensor], rel32: Optional[Tensor], wide: Optional[Tensor], time_thr: Tensor,
                   pos_table: Tensor, time_table: Optional[Tensor], num_heads: int, pos_bucket0: int) -> Tensor:
    """P [B, L, 4D] bf16 = [U | V | Q | K] -> O [B, L, D] bf16 = silu(Q K^T + bias) V, causal + key padding (hstu.py:244-267)."""
    require_cuda(P)
    B, L, D4 = P.shape
    D = D4 // 4
    has_time = time_table is not None and timestamps is not None
    dims = HstuDims(B, L, D, num_heads, pos_table.shape[0], time_table.shape[0] if has_time else 0, 0.0, 0, None, 0)
    O = torch.empty(B, L, D, dtype=torch.bfloat16, device=P.device)
    seq = _seq(pad, timestamps if has_time else None, rel32, wide, time_thr, pos_bucket0, dims.ntime)
    with torch.cuda.device(P.device):
        check(_lib.load().grb_hstu_attention_forward(C.byref(dims), ptr(pos_table), ptr(time_table) if has_time else None, C.byref(seq),
                                                     ptr(P.contiguous()), ptr(O), stream_ptr(P.device)))
    return O


@hstu_attention.register_fake
def _(P, pad, timestamps, rel32, wide, time_thr, pos_table, time_table, num_heads, pos_bucket0):
    B, L, D4 = P.shape
    return P.new_empty((B, L, D4 // 4))


@custom_op(f"{NS}::hstu_attention_backward", mutates_args=())
def hstu_attention_backward(P: Tensor, zp: Tensor, dO: Tensor, pad: Tensor, timestamps: Optional[Tensor], rel32: Optional[Tensor],
                            wide: Optional[Tensor], time_thr: Tensor, pos_table: Tensor, time_table: Optional[Tensor], num_heads: int,
                            pos_bucket0: int) -> Tuple[Tensor, Tensor, Tensor]:
    """-> dzp [B, L, 4D] bf16 (gradient w.r.t. the PRE-activations zp, columns V, Q, K; U = 0), dpos_table, dtime_table (fp32)."""
    B, L, D4 = P.shape
    D = D4 // 4
    has_time = time_table is not None and timestamps is not None
    dims = HstuDims(B, L, D, num_heads, pos_table.shape[0], time_table.shape[0] if has_time else 0, 0.0, 0, None, 0)
    lib = _lib.load()
    dzp = torch.zeros(B, L, D4, dtype=torch.bfloat16, device=P.device)
    dpos = torch.zeros(pos_table.shape, dtype=torch.float32, device=P.device)
    dtime = torch.zeros(time_table.shape if time_table is not None else (0, num_heads), dtype=torch.float32, device=P.device)
    scratch = torch.empty(lib.grb_hstu_attention_scratch_bytes(C.byref(dims)), dtype=torch.uint8, device=P.device)
    seq = _seq(pad, timestamps if has_time else None, rel32, wide, time_thr, pos_bucket0, dims.ntime)
    with torch.cuda.device(P.device):
        check(lib.grb_hstu_attention_backward(C.byref(dims), ptr(pos_table), ptr(time_table) if has_time else None, C.byref(seq),
                                              ptr(P.contiguous()), ptr(zp.contiguous()), ptr(dO.contiguous()), ptr(dzp), ptr(dpos),
                                              ptr(dtime) if has_time else None, ptr(scratch), stream_ptr(P.device)))
    return dzp, dpos, dtime


@hstu_attention_backward.register_fake
def _(P, zp, dO, pad, timestamps, rel32, wide, time_thr, pos_table, time_table, num_heads, pos_bucket0):
    tshape = time_table.shape if time_table is not None else (0, num_heads)
    return P.new_empty(P.shape), pos_table.new_empty(pos_table.shape, dtype=torch.float32), pos_table.new_empty(tshape, dtype=torch.float32)


# ------------------------------------------------------------------------------------------------ the whole block
_PNAMES = ("proj_w", "proj_b", "pos_table", "time_table", "ln1_g", "ln1_b", "ffn1_w", "ffn1_b", "ffn2_w", "ffn2_b", "ln2_g", "ln2_b")


def _layer_structs(x, pad, timestamps, rel32, wide, time_thr, params: List[Optional[Tensor]], bf16w: List[Tensor], H, ntime, pos_bucket0, p, seed,
                   seed_dev, layer):
    B, L, D = x.shape
    named = dict(zip(_PNAMES, params))
    has_time = named["time_table"] is not None and timestamps is not None
    dims = HstuDims(B, L, D, H, named["pos_table"].shape[0], ntime if has_time else 0, float(p), int(seed) & (2 ** 64 - 1), ptr(seed_dev), layer)
    bw = dict(zip(("proj_w", "ffn1_w", "ffn2_w"), bf16w))
    ps = HstuLayerParams(*[ptr(bw[n]) if n in bw else (ptr(named[n]) if named[n] is not None and (n != "time_table" or has_time) else None)
                           for n in _PNAMES])
    return dims, ps, _seq(pad, timestamps if has_time else None, rel32, wide, time_thr, pos_bucket0, dims.ntime), named, has_time


@custom_op(f"{NS}::hstu_layer", mutates_args=())
def hstu_layer(x: Tensor, pad: Tensor, timestamps: Optional[Tensor], rel32: Optional[Tensor], wide: Optional[Tensor], time_thr: Tensor,
               proj_w: Tensor, proj_b: Tensor, pos_table: Tensor, time_table: Optional[Tensor], ln1_g: Tensor, ln1_b: Tensor, ffn1_w: Tensor,
               ffn1_b: Tensor, ffn2_w: Tensor, ffn2_b: Tensor, ln2_g: Tensor, ln2_b: Tensor, num_heads: int, ntime: int, pos_bucket0: int,
               dropout_p: float, seed: int, seed_dev: Optional[Tensor], layer_index: int) -> Tuple[Tensor, Tensor]:
    """One HSTU block (hstu.py:222-280): x [B, L, D] fp32 -> (y [B, L, D] fp32, saved-for-backward blob uint8).  fp32 master
    weights in; the bf16 operand copies are made inside (one cast kernel each)."""
    require_cuda(x)
    lib = _lib.load()
    params = [proj_w, proj_b, pos_table, time_table, ln1_g, ln1_b, ffn1_w, ffn1_b, ffn2_w, ffn2_b, ln2_g, ln2_b]
    bf16w = [Fn.cast_bf16(w) for w in (proj_w, ffn1_w, ffn2_w)]
    xc = x.contiguous().float()
    dims, ps, seq, _, _ = _layer_structs(xc, pad, timestamps, rel32, wide, time_thr, params, bf16w, num_heads, ntime, pos_bucket0, dropout_p, seed,
                                         seed_dev, layer_index)
    nbytes = lib.grb_hstu_layer_saved_bytes(C.byref(dims))
    if nbytes == 0:
        raise _lib.GrbError(lib.grb_last_error().decode())
    saved = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    y = torch.empty_like(xc)
    with torch.cuda.device(x.device):
        check(lib.grb_hstu_layer_forward(C.byref(dims), C.byref(ps), C.byref(seq), ptr(xc), ptr(y), ptr(saved), stream_ptr(x.device)))
    return y, saved


def _saved_bytes(B, L, D):
    T = B * L
    al = lambda n: (n + 255) // 256 * 256
    return sum(al(n) for n in (T * D * 2, T * 4 * D * 2, T * 4 * D * 2, T * D * 2, T * 8, T * D * 4, T * D * 2, T * 8, T * 4 * D * 2, T * 4 * D * 2))


@hstu_layer.register_fake
def _(x, pad, timestamps, rel32, wide, time_thr, proj_w, proj_b, pos_table, time_table, ln1_g, ln1_b, ffn1_w, ffn1_b, ffn2_w, ffn2_b, ln2_g, ln2_b,
      num_heads, ntime, pos_bucket0, dropout_p, seed, seed_dev, layer_index):
    B, L, D = x.shape
    return x.new_empty(x.shape, dtype=torch.float32), x.new_empty((_saved_bytes(B, L, D),), dtype=torch.uint8)


@custom_op(f"{NS}::hstu_layer_backward", mutates_args=())
def hstu_layer_backward(dy: Tensor, saved: Tensor, pad: Tensor, timestamps: Optional[Tensor], rel32: Optional[Tensor], wide: Optional[Tensor],
                        time_thr: Tensor, proj_w: Tensor, proj_b: Tensor, pos_table: Tensor, time_table: Optional[Tensor], ln1_g: Tensor,
                        ln1_b: Tensor, ffn1_w: Tensor, ffn1_b: Tensor, ffn2_w: Tensor, ffn2_b: Tensor, ln2_g: Tensor, ln2_b: Tensor,
                        num_heads: int, ntime: int, pos_bucket0: int, dropout_p: float, seed: int, seed_dev: Optional[Tensor],
                        layer_index: int) -> List[Tensor]:
    """-> [dx, d proj_w, d proj_b, d pos_table, d time_table, d ln1_g, d ln1_b, d ffn1_w, d ffn1_b, d ffn2_w, d ffn2_b, d ln2_g, d ln2_b]
    (fp32; d time_table is an empty [0, H] tensor when the block has no temporal bias)."""
    lib = _lib.load()
    params = [proj_w, proj_b, pos_table, time_table, ln1_g, ln1_b, ffn1_w, ffn1_b, ffn2_w, ffn2_b, ln2_g, ln2_b]
    bf16w = [Fn.cast_bf16(w) for w in (proj_w, ffn1_w, ffn2_w)]
    dyc = dy.contiguous().float()
    dims, ps, seq, named, has_time = _layer_structs(dyc, pad, timestamps, rel32, wide, time_thr, params, bf16w, num_heads, ntime, pos_bucket0,
                                                    dropout_p, seed, seed_dev, layer_index)
    grads = {n: (torch.zeros(named[n].shape, dtype=torch.float32, device=dy.device) if named[n] is not None else None) for n in _PNAMES}
    gs = HstuLayerGrads(*[ptr(grads[n]) for n in _PNAMES])
    dx = torch.empty_like(dyc)
    ws = torch.empty(lib.grb_hstu_layer_workspace_bytes(C.byref(dims)), dtype=torch.uint8, device=dy.device)
    with torch.cuda.device(dy.device):
        check(lib.grb_hstu_layer_backward(C.byref(dims), C.byref(ps), C.byref(seq), ptr(dyc), ptr(saved), ptr(dx), C.byref(gs), ptr(ws),
                                          stream_ptr(dy.device)))
    out = [dx]
    for n in _PNAMES:
        out.append(grads[n] if grads[n] is not None else torch.zeros(0, num_heads, dtype=torch.float32, device=dy.device))
    return out


@hstu_layer_backward.register_fake
def _(dy, saved, pad, timestamps, rel32, wide, time_thr, proj_w, proj_b, pos_table, time_table, ln1_g, ln1_b, ffn1_w, ffn1_b, ffn2_w, ffn2_b, ln2_g,
      ln2_b, num_heads, ntime, pos_bucket0, dropout_p, seed, seed_dev, layer_index):
    ps = [proj_w, proj_b, pos_table, time_table, ln1_g, ln1_b, ffn1_w, ffn1_b, ffn2_w, ffn2_b, ln2_g, ln2_b]
    return [dy.new_empty(dy.shape, dtype=torch.float32)] + [
        (dy.new_empty(q.shape, dtype=torch.float32) if q is not None else dy.new_empty((0, num_heads), dtype=torch.float32)) for q in ps]


def _layer_setup(ctx, inputs, output):
    (x, pad, ts, rel32, wide, thr, *params, H, ntime, pb0, p, seed, seed_dev, layer) = inputs
    ctx.save_for_backward(output[1], pad, ts, rel32, wide, thr, *[q for q in params if q is not None], *([seed_dev] if seed_dev is not None else []))
    ctx.present = [q is not None for q in params]
    ctx.has = (ts is not None, rel32 is not None, wide is not None, seed_dev is not None)
    ctx.scalars = (H, ntime, pb0, p, seed, layer)


def _layer_backward(ctx, dy, _dsaved):
    it = iter(ctx.saved_tensors)
    saved, pad = next(it), next(it)
    ts, rel32, wide = next(it), next(it), next(it)       # saved as None when absent
    thr = next(it)
    params = [next(it) if pr else None for pr in ctx.present]
    seed_dev = next(it) if ctx.has[3] else None
    H, ntime, pb0, p, seed, layer = ctx.scalars
    g = torch.ops.genrec_b200.hstu_layer_backward(dy, saved, pad, ts, rel32, wide, thr, *params, H, ntime, pb0, p, seed, seed_dev, layer)
    pg = [g[1 + i] if pr else None for i, pr in enumerate(ctx.present)]
    return (g[0], None, None, None, None, None, *pg, None, None, None, None, None, None, None)


torch.library.register_autograd(f"{NS}::hstu_layer", _layer_backward, setup_context=_layer_setup)


# ------------------------------------------------------------------------------------------------ RQ-VAE search, metrics
@custom_op(f"{NS}::rq_residual_argmin", mutates_args=())
def rq_residual_argmin(x: Tensor, codebooks: Tensor, commitment: float) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """x [N, D] fp32, codebooks [levels, K, D] -> ids [N, levels] int64, emb / res [N, D, levels], loss [N] (rqvae.py:185-199, :397-412)."""
    ids, emb, res, loss = Fn.rq_residual_argmin(x, codebooks, commitment, want_aux=True)
    return ids, emb, res, loss


@rq_residual_argmin.register_fake
def _(x, codebooks, commitment):
    N, D = x.shape
    lv = codebooks.shape[0]
    return (x.new_empty((N, lv), dtype=torch.int64), x.new_empty((N, D, lv), dtype=torch.float32), x.new_empty((N, D, lv), dtype=torch.float32),
            x.new_empty((N,), dtype=torch.float32))


@custom_op(f"{NS}::rq_sinkhorn", mutates_args=())
def rq_sinkhorn(dist: Tensor, eps: float, iters: int) -> Tuple[Tensor, Tensor, Tensor]:
    """dist [B, K] fp32 -> Sinkhorn-Knopp hard ids [B] int64 and the final scalings u [B], v [K] fp64 (rqvae.py:85-110, :218-241)."""
    return Fn.rq_sinkhorn(dist, eps, iters)


@rq_sinkhorn.register_fake
def _(dist, eps, iters):
    B, K = dist.shape
    return dist.new_empty((B,), dtype=torch.int64), dist.new_empty((B,), dtype=torch.float64), dist.new_empty((K,), dtype=torch.float64)


@custom_op(f"{NS}::eval_rank_metrics", mutates_args=())
def eval_rank_metrics(logits_last: Tensor, targets: Tensor) -> Tensor:
    """[B, C] fp32 logits of the last position, targets [B] -> [6] fp32: Recall@{1,5,10} hit counts, NDCG@{1,5,10} sums."""
    return Fn.eval_rank_metrics(logits_last, targets)


@eval_rank_metrics.register_fake
def _(logits_last, targets):
    return logits_last.new_empty((6,), dtype=torch.float32)


# ------------------------------------------------------------------------------------------------ SASRec attention core
@custom_op(f"{NS}::sasrec_attention", mutates_args=())
def sasrec_attention(q: Tensor, k: Tensor, v: Tensor, pad: Tensor, num_heads: int, dropout_p: float, seed: int, seed_dev: Optional[Tensor],
                     layer_index: int) -> Tuple[Tensor, Tensor]:
    """q, k, v [B, L, D] bf16, pad [B, L] uint8 -> (softmax(mask(q k^T / sqrt(dh))) * query_mask) v [B, L, D] bf16, lse [B, H, L]
    (sasrec.py:205-239)."""
    return Fn.sasrec_attention_fwd(q.contiguous(), k.contiguous(), v.contiguous(), pad.contiguous(), num_heads, dropout_p, seed, seed_dev, layer_index)


@sasrec_attention.register_fake
def _(q, k, v, pad, num_heads, dropout_p, seed, seed_dev, layer_index):
    B, L, D = q.shape
    return q.new_empty(q.shape), q.new_empty((B, num_heads, L), dtype=torch.float32)


@custom_op(f"{NS}::sasrec_attention_backward", mutates_args=())
def sasrec_attention_backward(q: Tensor, k: Tensor, v: Tensor, pad: Tensor, out: Tensor, lse: Tensor, dout: Tensor, num_heads: int,
                              dropout_p: float, seed: int, seed_dev: Optional[Tensor], layer_index: int) -> Tuple[Tensor, Tensor, Tensor]:
    return Fn.sasrec_attention_bwd(q.contiguous(), k.contiguous(), v.contiguous(), pad.contiguous(), out.contiguous(), lse.contiguous(),
                                   dout.contiguous(), num_heads, dropout_p, seed, seed_dev, layer_index)


@sasrec_attention_backward.register_fake
def _(q, k, v, pad, out, lse, dout, num_heads, dropout_p, seed, seed_dev, layer_index):
    return q.new_empty(q.shape), q.new_empty(q.shape), q.new_empty(q.shape)


def _sas_setup(ctx, inputs, output):
    q, k, v, pad, H, p, seed, seed_dev, layer = inputs
    ctx.save_for_backward(q, k, v, pad, output[0], output[1], *([seed_dev] if seed_dev is not None else []))
    ctx.has_sd = seed_dev is not None
    ctx.scalars = (H, p, seed, layer)


def _sas_backward(ctx, dout, _dlse):
    q, k, v, pad, out, lse, *rest = ctx.saved_tensors
    H, p, seed, layer = ctx.scalars
    dq, dk, dv = torch.ops.genrec_b200.sasrec_attention_backward(q, k, v, pad, out, lse, dout, H, p, seed, rest[0] if ctx.has_sd else None, layer)
    return dq, dk, dv, None, None, None, None, None, None


torch.library.register_autograd(f"{NS}::sasrec_attention", _sas_backward, setup_context=_sas_setup)


OPS = ("hstu_seq_prepare", "hstu_attention", "hstu_attention_backward", "hstu_layer", "hstu_layer_backward", "rq_residual_argmin",
       "rq_sinkhorn", "eval_rank_metrics", "sasrec_attention", "sasrec_attention_backward")
