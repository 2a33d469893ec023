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

from typing import List, Optional, Tuple

import torch
from torch import Tensor
from torch.library import custom_op

from . import functional as Fn
from ._lib import HstuDims, require_cuda

NS = "genrec_b200"


def _meta(pad: Tensor, ts: Optional[Tensor], thr: Tensor, pos_bucket0: int, ntime: int) -> Fn.SeqMeta:
    """Sequence metadata of one op call: uniform position buckets (bucket pos_bucket0), and the bias-index matrix built on the
    caller's stream even under the deferred schedule - the kernels that read it and the tensor's lifetime follow that stream."""
    return Fn.SeqMeta(pad, ts, None, thr, ntime, 1, (True, int(pos_bucket0)), may_defer=False)


# ------------------------------------------------------------------------------------------------ attention core
@custom_op(f"{NS}::hstu_attention", mutates_args=())
def hstu_attention(P: Tensor, pad: Tensor, timestamps: Optional[Tensor], time_thr: Tensor, pos_table: Tensor, time_table: Optional[Tensor],
                   num_heads: int, pos_bucket0: int) -> Tensor:
    """P [B, L, 4D] bf16 = [U | V | Q | K] -> O [B, L, D] bf16 = silu(Q K^T + bias) V, causal + key padding (hstu.py:244-267)."""
    require_cuda(P)
    ntime = time_table.shape[0] if time_table is not None else 0
    meta = _meta(pad, timestamps if time_table is not None else None, time_thr, pos_bucket0, ntime)
    return Fn.hstu_attention_fwd(P.contiguous(), meta, num_heads, pos_table, time_table, ntime)


@hstu_attention.register_fake
def _(P, pad, timestamps, time_thr, pos_table, time_table, num_heads, pos_bucket0):
    B, L, D4 = P.shape
    return P.new_empty((B, L, D4 // 4))


@custom_op(f"{NS}::hstu_attention_backward", mutates_args=())
def hstu_attention_backward(P: Tensor, zp: Tensor, dO: Tensor, pad: Tensor, timestamps: Optional[Tensor], time_thr: Tensor,
                            pos_table: Tensor, time_table: Optional[Tensor], num_heads: int, pos_bucket0: int) -> Tuple[Tensor, Tensor, Tensor]:
    """-> dzp [B, L, 4D] bf16 (gradient w.r.t. the PRE-activations zp, columns V, Q, K; U = 0), dpos_table, dtime_table (fp32)."""
    ntime = time_table.shape[0] if time_table is not None else 0
    meta = _meta(pad, timestamps if time_table is not None else None, time_thr, pos_bucket0, ntime)
    dzp, dpos, dtime = Fn.hstu_attention_bwd(P.contiguous(), zp.contiguous(), dO.contiguous(), meta, num_heads, pos_table, time_table, ntime)
    if dtime is None:       # no temporal term: an all-zero gradient of the table, or [0, H] without one
        dtime = torch.zeros(time_table.shape if time_table is not None else (0, num_heads), dtype=torch.float32, device=P.device)
    return dzp, dpos, dtime


@hstu_attention_backward.register_fake
def _(P, zp, dO, pad, timestamps, time_thr, pos_table, time_table, num_heads, pos_bucket0):
    tshape = time_table.shape if time_table is not None else (0, num_heads)
    return P.new_empty(P.shape), pos_table.new_empty(pos_table.shape, dtype=torch.float32), pos_table.new_empty(tshape, dtype=torch.float32)


# ------------------------------------------------------------------------------------------------ the whole block
def _layer_call(shape, pad, timestamps, time_thr, params: List[Optional[Tensor]], H, ntime, pos_bucket0, p, seed, seed_dev, layer):
    """-> (dims, bf16 weight mirrors, has_time, meta) of one block op; params in Fn.PARAM_ORDER."""
    B, L, D = shape
    named = dict(zip(Fn.PARAM_ORDER, params))
    bf16w = {n: Fn.cast_bf16(named[n]) for n in Fn.BF16_PARAMS}
    has_time = named["time_table"] is not None and timestamps is not None
    dims = Fn._dims(B, L, D, H, named["pos_table"].shape[0], ntime if has_time else 0, p, seed, seed_dev, layer)
    return dims, bf16w, has_time, _meta(pad, timestamps if has_time else None, time_thr, pos_bucket0, dims.ntime)


@custom_op(f"{NS}::hstu_layer", mutates_args=())
def hstu_layer(x: Tensor, pad: Tensor, timestamps: Optional[Tensor], time_thr: Tensor, proj_w: Tensor, proj_b: Tensor, pos_table: Tensor,
               time_table: Optional[Tensor], ln1_g: Tensor, ln1_b: Tensor, ffn1_w: Tensor, ffn1_b: Tensor, ffn2_w: Tensor, ffn2_b: Tensor,
               ln2_g: Tensor, ln2_b: Tensor, num_heads: int, ntime: int, pos_bucket0: int, dropout_p: float, seed: int,
               seed_dev: Optional[Tensor], layer_index: int) -> Tuple[Tensor, Tensor]:
    """One HSTU block (hstu.py:222-280): x [B, L, D] fp32 -> (y [B, L, D] fp32, saved-for-backward blob uint8).  fp32 master
    weights in; the bf16 operand copies are made inside (one cast kernel each)."""
    require_cuda(x)
    params = [proj_w, proj_b, pos_table, time_table, ln1_g, ln1_b, ffn1_w, ffn1_b, ffn2_w, ffn2_b, ln2_g, ln2_b]
    dims, bf16w, has_time, meta = _layer_call(x.shape, pad, timestamps, time_thr, params, num_heads, ntime, pos_bucket0, dropout_p, seed,
                                              seed_dev, layer_index)
    return Fn.hstu_block_forward(dims, params, bf16w, has_time, meta, x.contiguous().float())


@hstu_layer.register_fake
def _(x, pad, timestamps, time_thr, proj_w, proj_b, pos_table, time_table, ln1_g, ln1_b, ffn1_w, ffn1_b, ffn2_w, ffn2_b, ln2_g, ln2_b,
      num_heads, ntime, pos_bucket0, dropout_p, seed, seed_dev, layer_index):
    B, L, D = x.shape
    nbytes = Fn.layer_saved_bytes(HstuDims(B, L, D, num_heads, pos_table.shape[0], 0, 0.0, 0, None, 0))   # depends on B, L, D only
    return x.new_empty(x.shape, dtype=torch.float32), x.new_empty((nbytes,), dtype=torch.uint8)


@custom_op(f"{NS}::hstu_layer_backward", mutates_args=())
def hstu_layer_backward(dy: Tensor, saved: Tensor, pad: Tensor, timestamps: Optional[Tensor], time_thr: Tensor, proj_w: Tensor,
                        proj_b: Tensor, pos_table: Tensor, time_table: Optional[Tensor], ln1_g: Tensor, ln1_b: Tensor, ffn1_w: Tensor,
                        ffn1_b: Tensor, ffn2_w: Tensor, ffn2_b: Tensor, ln2_g: Tensor, ln2_b: Tensor, num_heads: int, ntime: int,
                        pos_bucket0: int, dropout_p: float, seed: int, seed_dev: Optional[Tensor], layer_index: int) -> List[Tensor]:
    """-> [dx, d proj_w, d proj_b, d pos_table, d time_table, d ln1_g, d ln1_b, d ffn1_w, d ffn1_b, d ffn2_w, d ffn2_b, d ln2_g, d ln2_b]
    (fp32; d time_table is an empty [0, H] tensor when the block has no temporal bias)."""
    params = [proj_w, proj_b, pos_table, time_table, ln1_g, ln1_b, ffn1_w, ffn1_b, ffn2_w, ffn2_b, ln2_g, ln2_b]
    dims, bf16w, has_time, meta = _layer_call(dy.shape, pad, timestamps, time_thr, params, num_heads, ntime, pos_bucket0, dropout_p, seed,
                                              seed_dev, layer_index)
    dx, grads = Fn.hstu_block_backward(dims, params, bf16w, has_time, meta, dy, saved)
    return [dx] + [g if g is not None else torch.zeros(0, num_heads, dtype=torch.float32, device=dy.device) for g in grads]


@hstu_layer_backward.register_fake
def _(dy, saved, pad, timestamps, time_thr, proj_w, proj_b, pos_table, time_table, ln1_g, ln1_b, ffn1_w, ffn1_b, ffn2_w, ffn2_b, ln2_g, ln2_b,
      num_heads, ntime, pos_bucket0, dropout_p, seed, seed_dev, layer_index):
    ps = [proj_w, proj_b, pos_table, time_table, ln1_g, ln1_b, ffn1_w, ffn1_b, ffn2_w, ffn2_b, ln2_g, ln2_b]
    return [dy.new_empty(dy.shape, dtype=torch.float32)] + [
        (dy.new_empty(q.shape, dtype=torch.float32) if q is not None else dy.new_empty((0, num_heads), dtype=torch.float32)) for q in ps]


def _layer_setup(ctx, inputs, output):
    (x, pad, ts, thr, *params, H, ntime, pb0, p, seed, seed_dev, layer) = inputs
    ctx.save_for_backward(output[1], pad, ts, thr, *[q for q in params if q is not None], *([seed_dev] if seed_dev is not None else []))
    ctx.present = [q is not None for q in params]
    ctx.has_sd = seed_dev is not None
    ctx.scalars = (H, ntime, pb0, p, seed, layer)


def _layer_backward(ctx, dy, _dsaved):
    it = iter(ctx.saved_tensors)
    saved, pad = next(it), next(it)
    ts = next(it)       # saved as None when absent
    thr = next(it)
    params = [next(it) if pr else None for pr in ctx.present]
    seed_dev = next(it) if ctx.has_sd else None
    H, ntime, pb0, p, seed, layer = ctx.scalars
    g = torch.ops.genrec_b200.hstu_layer_backward(dy, saved, pad, ts, thr, *params, H, ntime, pb0, p, seed, seed_dev, layer)
    pg = [g[1 + i] if pr else None for i, pr in enumerate(ctx.present)]
    return (g[0], None, None, None, *pg, None, None, None, None, None, None, None)


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


@custom_op(f"{NS}::head_topk", mutates_args=())
def head_topk(x: Tensor, ln_g: Tensor, ln_b: Tensor, table_bf16: Tensor, eps: float, k: int, exclude: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
    """x [R, D] fp32 -> (scores [R, k] fp32, items [R, k] int64): the k best items of LN(x) E^T without the logits, item 0 and the
    row's exclude ids [R, E] int64 left out, ties to the lower id (hstu.py:150-157 for serving).  Inference only."""
    return tuple(Fn.head_topk(x, ln_g, ln_b, table_bf16, eps, k, exclude))


@head_topk.register_fake
def _(x, ln_g, ln_b, table_bf16, eps, k, exclude):
    R = x.shape[0]
    return x.new_empty((R, k), dtype=torch.float32), x.new_empty((R, k), dtype=torch.int64)


@custom_op(f"{NS}::head_candidates", mutates_args=())
def head_candidates(x: Tensor, ln_g: Tensor, ln_b: Tensor, table_bf16: Tensor, eps: float, k: int,
                    exclude: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
    """head_topk for up to 2048 items per row: x [R, D] fp32 -> (scores [R, k] fp32, items [R, k] int64), 1 <= k <= 2048, the
    same selection rules, without the logits.  Inference only."""
    return tuple(Fn.head_candidates(x, ln_g, ln_b, table_bf16, eps, k, exclude))


@head_candidates.register_fake
def _(x, ln_g, ln_b, table_bf16, eps, k, exclude):
    R = x.shape[0]
    return x.new_empty((R, k), dtype=torch.float32), x.new_empty((R, k), dtype=torch.int64)


@custom_op(f"{NS}::head_rank_metrics", mutates_args=())
def head_rank_metrics(x: Tensor, ln_g: Tensor, ln_b: Tensor, table_bf16: Tensor, eps: float, targets: Tensor,
                      exclude: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
    """x [R, D] fp32, targets [R] int64 -> (metrics [6] fp32, ranks [R] int32): eval_rank_metrics of the head's logits, counted
    without forming them; the row's exclude ids [R, E] int64 are left out of the count.  Inference only."""
    return tuple(Fn.head_rank_metrics(x, ln_g, ln_b, table_bf16, eps, targets, exclude=exclude, want_ranks=True))


@head_rank_metrics.register_fake
def _(x, ln_g, ln_b, table_bf16, eps, targets, exclude):
    return x.new_empty((6,), dtype=torch.float32), x.new_empty((x.shape[0],), dtype=torch.int32)


# ------------------------------------------------------------------------------------------------ sampled-softmax head
@custom_op(f"{NS}::head_sampled_loss", mutates_args=())
def head_sampled_loss(x: Tensor, ln_g: Tensor, ln_b: Tensor, table: Tensor, targets: Tensor, negatives: Tensor, log_q: Optional[Tensor],
                      eps: float) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """x [T, D] fp32, table [C, D] fp32, targets [T] (0 = ignored), negatives [N] shared by every token, log_q [C] or None ->
    (loss, dx [T, D], dln_g [D], dln_b [D], dtable [C, D]): the sampled softmax with logQ correction and, from the same pass, its
    gradients for a unit gradient of the loss (the autograd formula scales them)."""
    require_cuda(x)
    xc = x.contiguous().float()
    dx = torch.empty_like(xc)
    dtable = torch.zeros(table.shape, dtype=torch.float32, device=x.device)
    dg = torch.zeros(ln_g.shape, dtype=torch.float32, device=x.device)
    db = torch.zeros(ln_b.shape, dtype=torch.float32, device=x.device)
    loss = Fn.head_sampled_loss_raw(xc, ln_g, ln_b, Fn.cast_bf16(table), targets.contiguous(), negatives, log_q, eps, (dx, dtable, dg, db))
    return loss, dx, dg, db, dtable


@head_sampled_loss.register_fake
def _(x, ln_g, ln_b, table, targets, negatives, log_q, eps):
    f32 = dict(dtype=torch.float32)
    return (x.new_empty((), **f32), x.new_empty(x.shape, **f32), x.new_empty(ln_g.shape, **f32), x.new_empty(ln_b.shape, **f32),
            x.new_empty(table.shape, **f32))


def _sampled_setup(ctx, inputs, output):
    ctx.save_for_backward(*output[1:])


def _sampled_backward(ctx, dloss, *_):
    dx, dg, db, dtable = ctx.saved_tensors
    return dx * dloss, dg * dloss, db * dloss, dtable * dloss, None, None, None, None


torch.library.register_autograd(f"{NS}::head_sampled_loss", _sampled_backward, setup_context=_sampled_setup)


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


OPS = ("hstu_attention", "hstu_attention_backward", "hstu_layer", "hstu_layer_backward", "rq_residual_argmin", "rq_sinkhorn",
       "eval_rank_metrics", "head_topk", "head_candidates", "head_rank_metrics", "head_sampled_loss", "sasrec_attention",
       "sasrec_attention_backward")
