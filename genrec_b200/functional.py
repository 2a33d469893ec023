"""torch-facing wrappers of the C ABI: tensors in, tensors out, autograd wired by hand.

Every function here hands raw device pointers + the current CUDA stream to ``libgenrec_b200.so`` (ctypes, see
``_lib.py``); PyTorch only provides memory, streams and the autograd graph.  CPU tensors raise - there is no fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import List, Optional, Tuple

import torch

from . import _lib
from ._lib import HstuDims, HstuLayerGrads, HstuLayerParams, HstuSeq, SasrecDims, check, ptr, require_cuda, stream_ptr

PARAM_ORDER = ("proj_w", "proj_b", "pos_table", "time_table", "ln1_g", "ln1_b", "ffn1_w", "ffn1_b", "ffn2_w", "ffn2_b",
               "ln2_g", "ln2_b")
BF16_PARAMS = ("proj_w", "ffn1_w", "ffn2_w")


def require_f32(*tensors) -> None:
    for t in tensors:
        if t is not None and t.dtype != torch.float32:
            raise _lib.GrbError(f"genrec_b200 error -1: parameters / activations must be float32 (got {t.dtype}); the kernels keep fp32 "
                                "masters and make their own bf16 operand copies")


def require_i64(*tensors) -> None:
    for t in tensors:
        if t is not None and t.dtype != torch.int64:
            raise _lib.GrbError(f"genrec_b200 error -1: ids / targets / timestamps must be int64 (got {t.dtype})")


# ---- deferred weight gradients (see grb_set_defer_weight_grads): operand buffers of GEMMs that run on the library's side stream
#      are parked here until join_deferred(), so the caching allocator cannot hand them to later kernels of the main stream
_DEFER = {"on": False, "c": False, "keep": []}


def set_defer_weight_grads(on: bool) -> None:
    """Policy switch (FlatAdam(defer_weight_grads=True)); the library-side flag is raised per call, only for calls whose gradients go
    to the flat gradient sink (nothing but the optimizer reads those before the join)."""
    _DEFER["on"] = bool(on)


def _defer_for_call(active: bool) -> bool:
    if _DEFER["c"] != active:
        check(_lib.load().grb_set_defer_weight_grads(1 if active else 0))
        _DEFER["c"] = active
    return active


def join_deferred(device) -> None:
    """Make the deferred dW / dE GEMMs visible to the current stream of `device` and release their operand buffers."""
    if _DEFER["c"] or _DEFER["keep"]:
        with torch.cuda.device(device):
            check(_lib.load().grb_join_deferred(stream_ptr(device)))
        _DEFER["keep"].clear()


def _u8(n, device):
    return torch.empty(n, dtype=torch.uint8, device=device)


def cast_bf16(src: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 -> bf16 copy with our own kernel (weights mirror)."""
    require_cuda(src)
    src = src.detach().contiguous()
    if out is None:
        out = torch.empty(src.shape, dtype=torch.bfloat16, device=src.device)
    require_f32(src)
    with torch.cuda.device(src.device):
        check(_lib.load().grb_cast_f32_to_bf16(ptr(src), ptr(out), src.numel(), stream_ptr(src.device)))
    return out


_ZERO_TABLES = {}


class SeqMeta:
    """Per-batch sequence metadata shared by all layers of one forward: the pad flags, the raw timestamps and the
    [B, L, ld] uint16 bias-index matrix the attention kernels read.  The per-sequence int32 rebasing of the timestamps
    (``grb_hstu_seq_prepare``) is made on demand for the bucket test hook."""

    def __init__(self, pad_u8: torch.Tensor, timestamps: Optional[torch.Tensor], pos_bucket: Optional[torch.Tensor],
                 time_thr: torch.Tensor, num_time_buckets: int = 64, num_pos_buckets: int = 32, pos_uniform=None,
                 may_defer: bool = True):
        # may_defer=False builds the index on the caller's stream even under the deferred schedule (the custom ops, whose
        # callers order and free everything by that stream); pos_bucket may be None when pos_uniform is given
        require_cuda(pad_u8)
        B, L = pad_u8.shape
        self.B, self.L = B, L
        self.pad = pad_u8.contiguous()
        if self.pad.dtype != torch.uint8:
            raise _lib.GrbError("genrec_b200 error -1: pad flags must be uint8")
        if timestamps is not None and timestamps.dtype != torch.int64:
            raise _lib.GrbError(f"genrec_b200 error -1: timestamps must be int64, got {timestamps.dtype}")
        self.timestamps = timestamps.contiguous() if timestamps is not None else None
        self.pos_bucket = pos_bucket
        self.time_thr = time_thr
        self.num_time_buckets, self.num_pos_buckets = num_time_buckets, num_pos_buckets
        if pos_uniform is None:        # (uniform?, bucket) - a host-side property of the [L] table, cached by the caller
            pb = pos_bucket.cpu()
            pos_uniform = (bool((pb == pb[0]).all()), int(pb[0]))
        self.pos_uniform, self.pos_bucket0 = pos_uniform
        self.ld = (L + 7) // 8 * 8
        self.rel32 = self.wide = None
        self._build_bias_index(may_defer)

    def _ensure_rel(self):
        if self.timestamps is None or self.rel32 is not None:
            return
        dev = self.pad.device
        self.rel32 = torch.empty(self.B, self.L, dtype=torch.int32, device=dev)
        self.wide = torch.empty(self.B, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            check(_lib.load().grb_hstu_seq_prepare(ptr(self.timestamps), ptr(self.pad), self.B, self.L, ptr(self.rel32), ptr(self.wide),
                                                   stream_ptr(dev)))

    def _build_bias_index(self, may_defer: bool):
        B, L, dev = self.B, self.L, self.pad.device
        self.bias_index = torch.empty(B, L, self.ld, dtype=torch.int16, device=dev)
        nt = self.num_time_buckets if self.timestamps is not None else 0
        if self.pos_uniform:      # collapse to one effective position bucket (see grb_hstu_seq.pos_uniform)
            key = (L, str(dev))
            if key not in _ZERO_TABLES:
                _ZERO_TABLES[key] = torch.zeros(L, dtype=torch.uint8, device=dev)
            pb_arg, npos_arg = _ZERO_TABLES[key], 1
        else:
            pb_arg, npos_arg = self.pos_bucket, self.num_pos_buckets
        # deferred schedule: built on the side stream, joined before the first attention launch
        _defer_for_call(_DEFER["on"] and may_defer)
        with torch.cuda.device(dev):
            check(_lib.load().grb_hstu_bias_index(ptr(self.timestamps), ptr(self.pad), ptr(self.time_thr), ptr(pb_arg), B, L,
                                                  npos_arg, nt, ptr(self.bias_index), self.ld, stream_ptr(dev)))

    def struct(self) -> HstuSeq:
        return HstuSeq(ptr(self.bias_index), self.ld, 1 if self.timestamps is not None else 0, 1 if self.pos_uniform else 0,
                       self.pos_bucket0, ptr(self.timestamps), ptr(self.pad), ptr(self.rel32), ptr(self.wide), ptr(self.time_thr))

    def bucket_bytes(self, num_time_buckets: Optional[int] = None) -> torch.Tensor:
        """[B, L, L] uint8: the time bucket (or 64 = masked) of every cell as the in-kernel bucket routine derives it from the
        rebased timestamps (test hook)."""
        nt = self.num_time_buckets if num_time_buckets is None else num_time_buckets
        out = torch.full((self.B, self.L, self.L), 255, dtype=torch.uint8, device=self.pad.device)
        self._ensure_rel()
        seq = self.struct()
        with torch.cuda.device(self.pad.device):
            check(_lib.load().grb_hstu_bucket_bytes_debug(C.byref(seq), self.B, self.L, nt if self.timestamps is not None else 0, ptr(out),
                                                          stream_ptr(self.pad.device)))
        return out


def _dims(B, L, D, H, npos, ntime, p, seed, seed_dev, layer) -> HstuDims:
    return HstuDims(B, L, D, H, npos, ntime, float(p), int(seed) & (2 ** 64 - 1), ptr(seed_dev), layer)


def _layer_param_struct(params, bf16w: dict, has_time: bool) -> HstuLayerParams:
    """``params`` in PARAM_ORDER (fp32 masters; time_table may be None), ``bf16w`` the bf16 mirrors of BF16_PARAMS.  The
    time table is passed only when the block uses the temporal term."""
    named = dict(zip(PARAM_ORDER, params))
    return HstuLayerParams(*[
        ptr(bf16w[n]) if n in BF16_PARAMS else (ptr(named[n].detach()) if named[n] is not None and (n != "time_table" or has_time) else None)
        for n in PARAM_ORDER])


def layer_saved_bytes(dims: HstuDims) -> int:
    """Size of the block's saved-for-backward blob (a host-side query: no device needed)."""
    lib = _lib.load()
    nbytes = lib.grb_hstu_layer_saved_bytes(C.byref(dims))
    if nbytes == 0:
        raise _lib.GrbError(lib.grb_last_error().decode())
    return nbytes


def hstu_block_forward(dims: HstuDims, params, bf16w: dict, has_time: bool, meta: SeqMeta, x: torch.Tensor):
    """One HSTU block (grb_hstu_layer_forward): x [B, L, D] fp32 contiguous -> (y, saved-for-backward blob)."""
    saved = _u8(layer_saved_bytes(dims), x.device)
    y = torch.empty_like(x)
    pstruct, seq = _layer_param_struct(params, bf16w, has_time), meta.struct()
    with torch.cuda.device(x.device):
        check(_lib.load().grb_hstu_layer_forward(C.byref(dims), C.byref(pstruct), C.byref(seq), ptr(x), ptr(y), ptr(saved),
                                                 stream_ptr(x.device)))
    return y, saved


def hstu_block_backward(dims: HstuDims, params, bf16w: dict, has_time: bool, meta: SeqMeta, dy: torch.Tensor, saved: torch.Tensor,
                        sink: Optional[dict] = None):
    """grb_hstu_layer_backward -> (dx, parameter gradients in PARAM_ORDER, None where a parameter is absent).  With a ``sink``
    (name -> view of the flat gradient buffer of genrec_b200.optim.FlatAdam) the gradients accumulate there, and the weight
    gradients follow the deferred schedule when it is on."""
    lib = _lib.load()
    if sink is not None:
        grads = [sink[n] if q is not None else None for n, q in zip(PARAM_ORDER, params)]
    else:
        grads = [torch.zeros(q.shape, dtype=torch.float32, device=dy.device) if q is not None else None for q in params]
    pstruct, gstruct, seq = _layer_param_struct(params, bf16w, has_time), HstuLayerGrads(*[ptr(g) for g in grads]), meta.struct()
    dyc = dy.contiguous().float()
    dx = torch.empty_like(dyc)
    ws = _u8(lib.grb_hstu_layer_workspace_bytes(C.byref(dims)), dy.device)
    deferred = _defer_for_call(_DEFER["on"] and sink is not None)
    with torch.cuda.device(dy.device):
        check(lib.grb_hstu_layer_backward(C.byref(dims), C.byref(pstruct), C.byref(seq), ptr(dyc), ptr(saved), ptr(dx), C.byref(gstruct),
                                          ptr(ws), stream_ptr(dy.device)))
    if deferred:
        _DEFER["keep"].append((ws, saved, dyc))     # still read by the deferred dW GEMM
    return dx, grads


class HstuLayerFn(torch.autograd.Function):
    """One HSTU block.  forward = grb_hstu_layer_forward, backward = grb_hstu_layer_backward."""

    @staticmethod
    def forward(ctx, x, meta: SeqMeta, cfg: dict, bf16w: dict, *params):
        # params in PARAM_ORDER (fp32 masters; time_table may be None)
        require_cuda(x)
        B, L, D = x.shape
        require_f32(*[q for q in params if q is not None])
        has_time = params[PARAM_ORDER.index("time_table")] is not None and meta.timestamps is not None
        dims = _dims(B, L, D, cfg["H"], cfg["npos"], cfg["ntime"] if has_time else 0, cfg["p"], cfg["seed"], cfg["seed_dev"],
                     cfg["layer"])
        y, ctx.saved_blob = hstu_block_forward(dims, params, bf16w, has_time, meta, x.detach().contiguous().float())
        ctx.meta, ctx.cfg, ctx.bf16w, ctx.has_time, ctx.dims = meta, cfg, bf16w, has_time, dims
        ctx.save_for_backward(*[p for p in params if p is not None])
        ctx.param_present = [p is not None for p in params]
        return y

    @staticmethod
    def backward(ctx, dy):
        it = iter(ctx.saved_tensors)
        params = [next(it) if present else None for present in ctx.param_present]
        sink = ctx.cfg.get("grad_sink")     # accumulate straight into the flat gradient buffer (genrec_b200.optim.FlatAdam)
        dx, grads = hstu_block_backward(ctx.dims, params, ctx.bf16w, ctx.has_time, ctx.meta, dy, ctx.saved_blob, sink)
        ctx.saved_blob = None
        if sink is not None:
            return (dx, None, None, None, *([None] * len(PARAM_ORDER)))
        return (dx, None, None, None, *grads)


class EmbedFn(torch.autograd.Function):
    """x = dropout(E[ids] * scale (+ pos)) ; also emits the uint8 pad flags."""

    @staticmethod
    def forward(ctx, ids, table, pos_table, scale, mask_pad_rows, p, seed, seed_dev, sink=None):
        lib = _lib.load()
        require_cuda(ids, table)
        require_i64(ids)
        require_f32(table, pos_table)
        ctx.sink = sink
        B, L = ids.shape
        D = table.shape[1]
        ids = ids.contiguous()
        x = torch.empty(B, L, D, dtype=torch.float32, device=ids.device)
        pad = torch.empty(B, L, dtype=torch.uint8, device=ids.device)
        with torch.cuda.device(ids.device):
            check(lib.grb_embed_forward(ptr(ids), ptr(table.detach()), ptr(pos_table.detach()) if pos_table is not None else None,
                                        ptr(x), ptr(pad), B, L, D, float(scale), int(mask_pad_rows), float(p), int(seed), ptr(seed_dev),
                                        stream_ptr(ids.device)))
        ctx.save_for_backward(ids)
        ctx.args = (table.shape, None if pos_table is None else pos_table.shape, scale, mask_pad_rows, p, seed, seed_dev)
        ctx.mark_non_differentiable(pad)
        return x, pad

    @staticmethod
    def backward(ctx, dx, _dpad):
        lib = _lib.load()
        (ids,) = ctx.saved_tensors
        tshape, pshape, scale, mask_pad_rows, p, seed, seed_dev = ctx.args
        B, L = ids.shape
        D = tshape[1]
        dx = dx.contiguous().float()
        if ctx.sink is not None:
            dtable, dpos = ctx.sink
        else:
            dtable = torch.zeros(tshape, dtype=torch.float32, device=dx.device)
            dpos = torch.zeros(pshape, dtype=torch.float32, device=dx.device) if pshape is not None else None
        order = torch.sort(ids.reshape(-1), stable=True).indices   # tokens grouped by id, in token order
        scratch = torch.empty(B * L, D, dtype=torch.float32, device=dx.device)
        with torch.cuda.device(dx.device):
            check(lib.grb_embed_backward(ptr(ids), ptr(order), ptr(dx), ptr(dtable), ptr(dpos), B, L, D, float(scale), int(mask_pad_rows), float(p),
                                         int(seed), ptr(seed_dev), ptr(scratch), stream_ptr(dx.device)))
        if ctx.sink is not None:
            return (None,) * 9
        return None, dtable, dpos, None, None, None, None, None, None


class HeadLossFn(torch.autograd.Function):
    """loss = CE(LN(x) @ E^T, targets, ignore_index=0).  The fused kernel produces the gradients in the same pass as the loss;
    ``backward`` scales them by the incoming gradient of the loss.

    ``sink = (dln_g, dln_b, dtable)`` are views of the flat gradient buffer (genrec_b200.optim.FlatAdam).  The sink is only
    ever touched in ``backward``: the head gradients wait in scratch tensors and are added as ``sink += dloss * grad`` - any
    loss scaling (gradient accumulation, a GradScaler) reaches the head and embedding gradients exactly as it reaches the
    layers through ``dx``, and a forward that is never back-propagated leaves the gradient buffer alone.
    ``unit_loss_grad=True`` (opt-in, ``FlatAdam(..., unit_loss_grad=True)``) is the fast path of a plain ``loss.backward()``:
    the kernels accumulate straight into the sink during this call and ``backward`` hands ``dx`` on unscaled; the contract
    (the loss is back-propagated exactly once, with gradient 1) is checked ON THE DEVICE in ``backward`` - a violation traps."""

    @staticmethod
    def forward(ctx, x, ln_g, ln_b, table, table_bf16, targets, eps, sink=None, unit_loss_grad=False):
        lib = _lib.load()
        require_cuda(x, table, targets)
        require_i64(targets)
        require_f32(ln_g, ln_b, table)
        B, L, D = x.shape
        T, Cn = B * L, table.shape[0]
        xc = x.detach().contiguous().float()
        tg = targets.contiguous()
        need_grad = any(ctx.needs_input_grad[:4])
        direct = need_grad and sink is not None and unit_loss_grad
        ctx.sink, ctx.direct = sink, direct
        loss = torch.empty((), dtype=torch.float32, device=x.device)   # zeroed on the device by the target-count kernel
        ws = _u8(lib.grb_head_workspace_bytes(T, D, Cn), x.device)
        if direct:
            dx = torch.empty_like(xc)
            dg, db, dtable = sink
        elif need_grad:
            dx = torch.empty_like(xc)
            dtable = torch.zeros(table.shape, dtype=torch.float32, device=x.device)
            dg = torch.zeros_like(ln_g, dtype=torch.float32)
            db = torch.zeros_like(ln_b, dtype=torch.float32)
        else:
            dx = dtable = dg = db = None
        deferred = _defer_for_call(_DEFER["on"] and direct)
        with torch.cuda.device(x.device):
            check(lib.grb_head_loss_forward_backward(ptr(xc), ptr(ln_g.detach()), ptr(ln_b.detach()), float(eps), ptr(table_bf16), ptr(tg),
                                                     T, D, Cn, ptr(loss), ptr(dx), ptr(dtable), ptr(dg), ptr(db), ptr(ws),
                                                     stream_ptr(x.device)))
        if deferred:
            _DEFER["keep"].append((ws, xc, tg))                   # xf, the shifts and the targets are still read by the deferred dE pass
        ctx.grads = (dx, dg, db, dtable)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        dx, dg, db, dtable = ctx.grads
        ctx.grads = None
        if dx is None:
            return (None,) * 9
        if ctx.direct:
            with torch.cuda.device(dx.device):
                check(_lib.load().grb_assert_unit_scalar(ptr(dloss.detach().float().contiguous()), stream_ptr(dx.device)))
            return dx, None, None, None, None, None, None, None, None
        if ctx.sink is not None:
            sg, sb, st = ctx.sink
            sg.add_(dg * dloss); sb.add_(db * dloss); st.addcmul_(dtable, dloss)
            return dx * dloss, None, None, None, None, None, None, None, None
        return dx * dloss, dg * dloss, db * dloss, dtable * dloss, None, None, None, None, None


def head_logits(x, ln_g, ln_b, table, table_bf16, eps) -> torch.Tensor:
    """fp32 logits [B, L, C] (no autograd - inference / API parity path)."""
    lib = _lib.load()
    require_cuda(x, table)
    B, L, D = x.shape
    T, Cn = B * L, table.shape[0]
    xc = x.detach().contiguous().float()
    logits = torch.empty(B, L, Cn, dtype=torch.float32, device=x.device)
    ws = _u8(lib.grb_head_workspace_bytes(T, D, Cn), x.device)
    with torch.cuda.device(x.device):
        check(lib.grb_head_logits(ptr(xc), ptr(ln_g.detach()), ptr(ln_b.detach()), float(eps), ptr(table_bf16), T, D, Cn, ptr(logits), ptr(ws),
                                  stream_ptr(x.device)))
    return logits


def eval_rank_metrics(logits_last: torch.Tensor, targets: torch.Tensor, metrics: Optional[torch.Tensor] = None,
                      want_ranks: bool = False):
    """logits_last [B, C] fp32, targets [B] int64 -> metrics [6] fp32 accumulated on the device:
    Recall@{1,5,10} hit counts, NDCG@{1,5,10} sums (hstu_trainer.py:55-81 without the per-sample host loop)."""
    require_cuda(logits_last, targets)
    require_i64(targets)
    lg = logits_last.detach().contiguous().float()
    B, Cn = lg.shape
    if metrics is None:
        metrics = torch.zeros(6, dtype=torch.float32, device=lg.device)
    ranks = torch.empty(B, dtype=torch.int32, device=lg.device) if want_ranks else None
    with torch.cuda.device(lg.device):
        check(_lib.load().grb_eval_rank_metrics(ptr(lg), ptr(targets.contiguous()), B, Cn, ptr(metrics), ptr(ranks), stream_ptr(lg.device)))
    return (metrics, ranks) if want_ranks else metrics


# ------------------------------------------------------------------------------------------------ attention core alone
def hstu_attention_fwd(P: torch.Tensor, meta: SeqMeta, H: int, pos_table: torch.Tensor, time_table: Optional[torch.Tensor],
                       ntime: int = 64) -> torch.Tensor:
    """P [B, L, 4D] bf16 = silu(x Wp^T + b) = [U | V | Q | K]  ->  O [B, L, D] bf16 (hstu.py:244-267)."""
    lib = _lib.load()
    require_cuda(P)
    B, L, D4 = P.shape
    D = D4 // 4
    has_time = time_table is not None and meta.timestamps is not None
    dims = _dims(B, L, D, H, pos_table.shape[0], ntime if has_time else 0, 0.0, 0, None, 0)
    O = torch.empty(B, L, D, dtype=torch.bfloat16, device=P.device)
    seq = meta.struct()
    with torch.cuda.device(P.device):
        check(lib.grb_hstu_attention_forward(C.byref(dims), ptr(pos_table), ptr(time_table) if has_time else None, C.byref(seq), ptr(P), ptr(O),
                                             stream_ptr(P.device)))
    return O


def hstu_attention_bwd(P, zp, dO, meta: SeqMeta, H: int, pos_table, time_table, ntime: int = 64):
    """-> dzp [B, L, 4D] bf16 (columns V, Q, K written; U untouched = 0), dpos_table, dtime_table (fp32)."""
    lib = _lib.load()
    B, L, D4 = P.shape
    D = D4 // 4
    has_time = time_table is not None and meta.timestamps is not None
    dims = _dims(B, L, D, H, pos_table.shape[0], ntime if has_time else 0, 0.0, 0, None, 0)
    dzp = torch.zeros(B, L, D4, dtype=torch.bfloat16, device=P.device)
    dpos = torch.zeros_like(pos_table, dtype=torch.float32)
    dtime = torch.zeros_like(time_table, dtype=torch.float32) if has_time else None
    scratch = _u8(lib.grb_hstu_attention_scratch_bytes(C.byref(dims)), P.device)
    seq = meta.struct()
    with torch.cuda.device(P.device):
        check(lib.grb_hstu_attention_backward(C.byref(dims), ptr(pos_table), ptr(time_table) if has_time else None, C.byref(seq), ptr(P), ptr(zp),
                                              ptr(dO), ptr(dzp), ptr(dpos), ptr(dtime), ptr(scratch), stream_ptr(P.device)))
    return dzp, dpos, dtime


# ------------------------------------------------------------------------------------------------ cached incremental inference
def hstu_cache_append(cache: _lib.HstuCache, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor]):
    """input_ids / timestamps [B, n] int64 -> (positions [B, n] int32, last_row [B] int32); advances the cache's lengths and stores
    the chunk's timestamps (grb_hstu_cache_append)."""
    require_cuda(input_ids, timestamps)
    require_i64(input_ids, timestamps)
    B, n = input_ids.shape
    positions = torch.empty(B, n, dtype=torch.int32, device=input_ids.device)
    last_row = torch.empty(B, dtype=torch.int32, device=input_ids.device)
    with torch.cuda.device(input_ids.device):
        check(_lib.load().grb_hstu_cache_append(C.byref(cache), ptr(input_ids.contiguous()),
                                                ptr(timestamps.contiguous()) if timestamps is not None else None, n, ptr(positions),
                                                ptr(last_row), stream_ptr(input_ids.device)))
    return positions, last_row


def hstu_layer_extend(x: torch.Tensor, cache, layer: int, positions: torch.Tensor, pos_bucket: Optional[torch.Tensor],
                      pos_bucket0: int, time_thr: torch.Tensor, H: int, npos: int, ntime: int, bf16w: dict, params,
                      users: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One block on a chunk against the cache: x [B, n, D] fp32 -> y [B, n, D] fp32.  ``cache`` is a dense ``HstuCache``
    (grb_hstu_layer_extend) or an ``HstuPool`` with ``users`` [B] int64 on the device (grb_hstu_layer_extend_paged).  ``params`` in
    PARAM_ORDER (time_table None or ntime = 0: no temporal term), ``bf16w`` the three bf16 weight mirrors."""
    lib = _lib.load()
    require_cuda(x)
    require_f32(x)
    B, n, D = x.shape
    xc = x.contiguous()
    has_time = params[PARAM_ORDER.index("time_table")] is not None and ntime > 0
    dims = _dims(B, n, D, H, npos, ntime if has_time else 0, 0.0, 0, None, layer)
    pstruct = _layer_param_struct(params, bf16w, has_time)
    paged = isinstance(cache, _lib.HstuPool)
    if paged:
        nbytes = lib.grb_hstu_layer_extend_paged_workspace_bytes(C.byref(dims), C.byref(cache))
    else:
        nbytes = lib.grb_hstu_layer_extend_workspace_bytes(C.byref(dims), cache.capacity)
    if nbytes == 0:
        raise _lib.GrbError(lib.grb_last_error().decode())
    ws = _u8(nbytes, x.device)
    y = torch.empty_like(xc)
    with torch.cuda.device(x.device):
        if paged:
            check(lib.grb_hstu_layer_extend_paged(C.byref(dims), C.byref(pstruct), C.byref(cache), layer, ptr(users), ptr(positions),
                                                  ptr(pos_bucket), int(pos_bucket0), ptr(time_thr), ptr(xc), ptr(y), ptr(ws),
                                                  stream_ptr(x.device)))
        else:
            check(lib.grb_hstu_layer_extend(C.byref(dims), C.byref(pstruct), C.byref(cache), layer, ptr(positions), ptr(pos_bucket),
                                            int(pos_bucket0), ptr(time_thr), ptr(xc), ptr(y), ptr(ws), stream_ptr(x.device)))
    return y


def hstu_pool_append(pool: _lib.HstuPool, users: torch.Tensor, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor]):
    """users [B] int64 and input_ids / timestamps [B, n] int64 on the device -> (positions [B, n] int32, last_row [B] int32, room [B]
    int32); hands out the pages the chunk needs and stores its timestamps (grb_hstu_pool_append)."""
    require_cuda(users, input_ids, timestamps)
    require_i64(users, input_ids, timestamps)
    B, n = input_ids.shape
    dev = input_ids.device
    positions = torch.empty(B, n, dtype=torch.int32, device=dev)
    last_row = torch.empty(B, dtype=torch.int32, device=dev)
    room = torch.empty(B, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        check(_lib.load().grb_hstu_pool_append(C.byref(pool), ptr(users.contiguous()), B, ptr(input_ids.contiguous()),
                                               ptr(timestamps.contiguous()) if timestamps is not None else None, n, ptr(positions),
                                               ptr(last_row), ptr(room), stream_ptr(dev)))
    return positions, last_row, room


def hstu_pool_release(pool: _lib.HstuPool, users: torch.Tensor, last_hidden: Optional[torch.Tensor]) -> None:
    """Return the pages of users [B] int64 (device) to the pool and zero their lengths, flags and rows of last_hidden [*, D] fp32."""
    require_cuda(users, last_hidden)
    require_i64(users)
    D = last_hidden.shape[1] if last_hidden is not None else 0
    with torch.cuda.device(users.device):
        check(_lib.load().grb_hstu_pool_release(C.byref(pool), ptr(users.contiguous()), users.numel(), ptr(last_hidden), D,
                                                stream_ptr(users.device)))


# ------------------------------------------------------------------------------------------------ SASRec pieces
def layernorm_fwd(x, g, b, eps, want_bf16=True, want_f32=False):
    lib = _lib.load()
    T, D = x.numel() // x.shape[-1], x.shape[-1]
    yb = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device) if want_bf16 else None
    yf = torch.empty(x.shape, dtype=torch.float32, device=x.device) if want_f32 else None
    st = torch.empty(T, 2, dtype=torch.float32, device=x.device)
    check(lib.grb_layernorm_forward(ptr(x), ptr(g), ptr(b), float(eps), T, D, ptr(yb), ptr(yf), ptr(st), stream_ptr(x.device)))
    return yb, yf, st


def layernorm_bwd(dy, x, st, g, residual=None):
    lib = _lib.load()
    T, D = x.numel() // x.shape[-1], x.shape[-1]
    dx = torch.empty_like(x)
    dg = torch.zeros_like(g)
    db = torch.zeros_like(g)
    ws = _u8(lib.grb_layernorm_backward_workspace_bytes(T, D), x.device)
    check(lib.grb_layernorm_backward(ptr(dy), ptr(x), ptr(st), ptr(g), ptr(residual), T, D, ptr(dx), ptr(dg), ptr(db), ptr(ws),
                                     stream_ptr(x.device)))
    return dx, dg, db


def linear_fwd(xb, wb, bias, act, p=0.0, seed=0, seed_dev=None, site=0):
    """z = xb @ wb^T + bias (bf16) ; act: 0 none, 1 silu, 2 relu -> returns (z, act(z) with dropout)"""
    lib = _lib.load()
    T, K = xb.numel() // xb.shape[-1], xb.shape[-1]
    N = wb.shape[0]
    z = torch.empty(*xb.shape[:-1], N, dtype=torch.bfloat16, device=xb.device)
    a = torch.empty_like(z) if act else None
    check(lib.grb_linear_forward(ptr(xb), ptr(wb), ptr(bias), T, N, K, act, ptr(z), ptr(a), float(p), int(seed), ptr(seed_dev), site,
                                 stream_ptr(xb.device)))
    return z, a


def linear_residual_fwd(xb, wb, bias, residual, row_scale=None, p=0.0, seed=0, seed_dev=None, site=0):
    lib = _lib.load()
    T, K = xb.numel() // xb.shape[-1], xb.shape[-1]
    N = wb.shape[0]
    y = torch.empty(*xb.shape[:-1], N, dtype=torch.float32, device=xb.device)
    check(lib.grb_linear_residual_forward(ptr(xb), ptr(wb), ptr(bias), ptr(residual), ptr(row_scale), T, N, K, ptr(y), float(p), int(seed),
                                          ptr(seed_dev), site, stream_ptr(xb.device)))
    return y


def linear_bwd(dyb, wb, xb, need_dx=True, dx_residual=None, need_dw=True):
    """dyb [T,N] bf16 ; wb [N,K] bf16 ; xb [T,K] bf16 -> dx fp32 [T,K] (+ residual), dw fp32 [N,K], db fp32 [N]"""
    lib = _lib.load()
    N, K = wb.shape
    T = dyb.numel() // N
    dx = torch.empty(*dyb.shape[:-1], K, dtype=torch.float32, device=dyb.device) if need_dx else None
    dw = torch.zeros(N, K, dtype=torch.float32, device=dyb.device) if need_dw else None
    db = torch.zeros(N, dtype=torch.float32, device=dyb.device) if need_dw else None
    ws = _u8(lib.grb_linear_backward_workspace_bytes(T, N, K), dyb.device) if need_dw else None
    check(lib.grb_linear_backward(ptr(dyb), ptr(wb), ptr(xb), T, N, K, ptr(dx), ptr(dx_residual), ptr(dw), ptr(db), ptr(ws),
                                  stream_ptr(dyb.device)))
    return dx, dw, db


def sasrec_attention_fwd(q, k, v, pad, H, p=0.0, seed=0, seed_dev=None, layer=0):
    lib = _lib.load()
    B, L, D = q.shape
    dims = SasrecDims(B, L, D, H, float(p), int(seed), ptr(seed_dev), layer)
    out = torch.empty_like(q)
    lse = torch.empty(B, H, L, dtype=torch.float32, device=q.device)
    check(lib.grb_sasrec_attention_forward(C.byref(dims), ptr(q), ptr(k), ptr(v), ptr(pad), ptr(out), ptr(lse), stream_ptr(q.device)))
    return out, lse


def sasrec_attention_bwd(q, k, v, pad, out, lse, dout, H, p=0.0, seed=0, seed_dev=None, layer=0):
    lib = _lib.load()
    B, L, D = q.shape
    dims = SasrecDims(B, L, D, H, float(p), int(seed), ptr(seed_dev), layer)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
    check(lib.grb_sasrec_attention_backward(C.byref(dims), ptr(q), ptr(k), ptr(v), ptr(pad), ptr(out), ptr(lse), ptr(dout), ptr(dq), ptr(dk),
                                            ptr(dv), stream_ptr(q.device)))
    return dq, dk, dv


def linear_dact_bwd(dyb, wb, z, act, p=0.0, seed=0, seed_dev=None, site=0):
    """g[T,K] = dropmask(dyb[T,N] @ wb[N,K]) * act'(z[T,K])  (bf16)"""
    N, K = wb.shape
    T = dyb.numel() // N
    g = torch.empty_like(z)
    check(_lib.load().grb_linear_dact_backward(ptr(dyb), ptr(wb), ptr(z), T, N, K, act, float(p), int(seed), ptr(seed_dev), site, ptr(g),
                                               stream_ptr(dyb.device)))
    return g


def cast_rows_bf16(x, row_scale=None, p=0.0, seed=0, seed_dev=None, site=0):
    """bf16(dropmask(x) * row_scale[:, None])"""
    D = x.shape[-1]
    T = x.numel() // D
    out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    check(_lib.load().grb_cast_rows_f32_to_bf16(ptr(x), ptr(out), T, D, ptr(row_scale), float(p), int(seed), ptr(seed_dev), site,
                                                stream_ptr(x.device)))
    return out


# ------------------------------------------------------------------------------------------------ RQ-VAE
def rq_residual_argmin(x: torch.Tensor, codebooks: torch.Tensor, commitment: float = 0.25, want_aux: bool = True):
    """x [N, D] fp32, codebooks [levels, K, D] fp32 -> ids [N, levels] int64 (+ emb, res [N, D, levels], loss [N])."""
    lib = _lib.load()
    require_cuda(x, codebooks)
    x = x.detach().contiguous().float()
    cb = codebooks.detach().contiguous().float()
    N, D = x.shape
    levels, K, _ = cb.shape
    if D not in (32, 64):
        raise _lib.GrbError(f"genrec_b200 error -1: latent dim {D} unsupported (32, 64)")
    ids = torch.empty(N, levels, dtype=torch.int64, device=x.device)
    emb = torch.empty(N, D, levels, dtype=torch.float32, device=x.device) if want_aux else None
    res = torch.empty(N, D, levels, dtype=torch.float32, device=x.device) if want_aux else None
    loss = torch.empty(N, dtype=torch.float32, device=x.device) if want_aux else None
    if N == 0:
        return ids, emb, res, loss
    with torch.cuda.device(x.device):
        check(lib.grb_rq_residual_argmin(ptr(x), ptr(cb), N, D, K, levels, float(commitment), ptr(ids), ptr(emb), ptr(res), ptr(loss), None,
                                         stream_ptr(x.device)))
    return ids, emb, res, loss


def rq_sinkhorn(dist: torch.Tensor, eps: float = 0.003, iters: int = 100):
    """Sinkhorn-Knopp hard assignment of the SINKHORN estimator (csrc/rq_sinkhorn.cuh): dist [B, K] fp32, 2 <= K <= 256 ->
    ids [B] int64, u [B] and v [K] fp64 (the final scalings; P = u K v)."""
    lib = _lib.load()
    require_cuda(dist)
    require_f32(dist)
    if dist.dim() != 2:
        raise _lib.GrbError(f"genrec_b200 error -1: dist must be [B, K] (got {tuple(dist.shape)})")
    dist = dist.detach().contiguous()
    B, K = dist.shape
    ids = torch.empty(B, dtype=torch.int64, device=dist.device)
    u = torch.empty(B, dtype=torch.float64, device=dist.device)
    v = torch.empty(K, dtype=torch.float64, device=dist.device)
    ws = _u8(lib.grb_rq_sinkhorn_workspace_bytes(B, K), dist.device)
    with torch.cuda.device(dist.device):
        check(lib.grb_rq_sinkhorn(ptr(dist), B, K, float(eps), int(iters), ptr(ids), ptr(u), ptr(v), ptr(ws), stream_ptr(dist.device)))
    return ids, u, v


def kmeans_update(x: torch.Tensor, assign: torch.Tensor, centroids: torch.Tensor) -> torch.Tensor:
    """One Lloyd update after the assignment (csrc/rq_sinkhorn.cuh kmeans_update_kernel): every non-empty cluster's centroid becomes
    the mean of its rows, in place.  Returns [2, k] int32: row 0 the cluster sizes, row 1 the centroid shifts (fp32 bits)."""
    require_cuda(x, assign, centroids)
    require_f32(x, centroids)
    require_i64(assign)
    if not centroids.is_contiguous():
        raise _lib.GrbError("genrec_b200 error -1: centroids must be contiguous (updated in place)")
    x = x.detach().contiguous()
    B, D = x.shape
    k = centroids.shape[0]
    stats = torch.empty(2, k, dtype=torch.int32, device=x.device)
    with torch.cuda.device(x.device):
        check(_lib.load().grb_kmeans_update(ptr(x), ptr(assign.contiguous()), B, D, k, ptr(centroids), ptr(stats[0]), ptr(stats[1]),
                                            stream_ptr(x.device)))
    return stats


def split3(x: torch.Tensor, operand: int) -> torch.Tensor:
    """fp32 [rows, K] -> bf16 [rows, 6K]: the three-term bf16 split of every value, laid out along K for the fp32-accurate GEMM
    (operand 0 = activation layout, 1 = weight layout; csrc/rowwise.cuh split3_f32_bf16_kernel)."""
    require_cuda(x)
    require_f32(x)
    x = x.detach().contiguous()
    rows, K = x.numel() // x.shape[-1], x.shape[-1]
    out = torch.empty(*x.shape[:-1], 6 * K, dtype=torch.bfloat16, device=x.device)
    with torch.cuda.device(x.device):
        check(_lib.load().grb_split3_f32_to_bf16(ptr(x), ptr(out), rows, K, operand, stream_ptr(x.device)))
    return out


def linear_f32x3(x_split: torch.Tensor, w_split: torch.Tensor, act: int = 0) -> torch.Tensor:
    """y = act(x W^T) in fp32 accuracy on the tensor-core path; x_split [T, 6K], w_split [N, 6K] from split3(); act 0 none, 1 silu."""
    K6 = x_split.shape[-1]
    T, N = x_split.numel() // K6, w_split.shape[0]
    y = torch.empty(*x_split.shape[:-1], N, dtype=torch.float32, device=x_split.device)
    with torch.cuda.device(x_split.device):
        check(_lib.load().grb_linear_f32x3_forward(ptr(x_split), ptr(w_split), T, N, K6 // 6, act, ptr(y), stream_ptr(x_split.device)))
    return y


def linear_f32x3_bias(x_split: torch.Tensor, w_split: torch.Tensor, bias: Optional[torch.Tensor], residual: Optional[torch.Tensor] = None,
                      act: int = 0) -> torch.Tensor:
    """y = act(x W^T + bias) + residual in fp32 accuracy; N need not be a multiple of 4 (the output pitch is padded and sliced)."""
    K6 = x_split.shape[-1]
    T, N = x_split.numel() // K6, w_split.shape[0]
    ldy = (N + 3) // 4 * 4
    if residual is not None and ldy != N:
        raise _lib.GrbError("genrec_b200 error -1: residual needs N % 4 == 0")
    y = torch.empty(*x_split.shape[:-1], ldy, dtype=torch.float32, device=x_split.device)
    with torch.cuda.device(x_split.device):
        check(_lib.load().grb_linear_f32x3_bias_forward(ptr(x_split), ptr(w_split), ptr(bias), ptr(residual), T, N, K6 // 6, act, ptr(y), ldy,
                                                        stream_ptr(x_split.device)))
    return y[..., :N] if ldy != N else y


def layernorm_f32(x: torch.Tensor, g: torch.Tensor, b: torch.Tensor, eps: float) -> torch.Tensor:
    require_cuda(x)
    require_f32(x, g, b)
    x = x.detach().contiguous()
    y = torch.empty_like(x)
    with torch.cuda.device(x.device):
        check(_lib.load().grb_layernorm_f32_forward(ptr(x), ptr(g.detach()), ptr(b.detach()), float(eps), x.numel() // x.shape[-1], x.shape[-1],
                                                    ptr(y), stream_ptr(x.device)))
    return y


def hstu_layer_forward_f32(x: torch.Tensor, meta: SeqMeta, H: int, npos: int, ntime: int, split_w: dict, params) -> torch.Tensor:
    """fp32-exact forward of one HSTU block (csrc/exact_f32.cuh; hstu.py:222-280 without autocast).  ``split_w`` = the three weight
    matrices pre-split by split3(w, 1); ``params`` in PARAM_ORDER.  Forward only."""
    require_cuda(x)
    require_f32(x)
    lib = _lib.load()
    B, L, D = x.shape
    xc = x.detach().contiguous()
    (_, proj_b, pos_t, time_t, ln1_g, ln1_b, _, ffn1_b, _, ffn2_b, ln2_g, ln2_b) = params
    join_deferred(x.device)
    seq = meta.struct()
    d = _dims(B, L, D, H, npos, ntime, 0.0, 0, None, 0)
    p = _lib.HstuLayerParamsF32(ptr(split_w["proj_w"]), ptr(proj_b.detach()), ptr(pos_t.detach()), ptr(time_t.detach()) if time_t is not None else None,
                                ptr(ln1_g.detach()), ptr(ln1_b.detach()), ptr(split_w["ffn1_w"]), ptr(ffn1_b.detach()), ptr(split_w["ffn2_w"]),
                                ptr(ffn2_b.detach()), ptr(ln2_g.detach()), ptr(ln2_b.detach()))
    ws = _u8(lib.grb_hstu_layer_f32_workspace_bytes(C.byref(d)), x.device)
    y = torch.empty_like(xc)
    with torch.cuda.device(x.device):
        check(lib.grb_hstu_layer_forward_f32(C.byref(d), C.byref(p), C.byref(seq), ptr(xc), ptr(y), ptr(ws), stream_ptr(x.device)))
    return y


def adam_step(p, g, m, v, p_bf16, state, lr, beta1, beta2, eps, weight_decay, grad_scale=1.0, zero_grad=True):
    with torch.cuda.device(p.device):
        check(_lib.load().grb_adam_step(ptr(p), ptr(g), ptr(m), ptr(v), ptr(p_bf16), p.numel(), ptr(state), lr, beta1, beta2, eps, weight_decay,
                                        grad_scale, int(zero_grad), stream_ptr(p.device)))
