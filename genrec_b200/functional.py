"""torch-facing wrappers of the C ABI: tensors in, tensors out, autograd wired by hand.

Every function here hands raw device pointers to ``libgenrec_b200.so`` through ``_lib.call``, which runs each launch under
its tensors' device and on that device's current stream; PyTorch only provides memory, streams and the autograd graph.  CPU
tensors raise - there is no fallback.
"""
from __future__ import annotations

import ctypes as C
import functools
import os
from typing import List, NamedTuple, Optional, Tuple

import torch

from . import _lib
from ._lib import HstuDims, HstuLayerGrads, HstuLayerParams, HstuSeq, SasrecDims, call, ensure_device, ptr, require_cuda, workspace

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
        _lib.defer_weight_grads(active)
        _DEFER["c"] = active
    return active


def join_deferred(device) -> None:
    """Make the deferred dW / dE GEMMs visible to the current stream of `device` and release their operand buffers."""
    if _DEFER["c"] or _DEFER["keep"]:
        call(device, "grb_join_deferred")
        _DEFER["keep"].clear()


def cast_bf16(src: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fp32 -> bf16 copy with our own kernel (weights mirror)."""
    require_cuda(src)
    src = src.detach().contiguous()
    if out is None:
        out = torch.empty(src.shape, dtype=torch.bfloat16, device=src.device)
    require_f32(src)
    call(src.device, "grb_cast_f32_to_bf16", ptr(src), ptr(out), src.numel())
    return out


_ZERO_TABLES = {}


class SeqMeta:
    """Per-batch sequence metadata shared by all layers of one forward: the pad flags, the raw timestamps and the
    [B, L, ld] uint16 bias-index matrix the attention kernels read.  With ``offsets`` ([B+1] int64 on the device) and
    ``max_len`` the batch is packed: pad_u8 / timestamps are [T] and the index matrix is [T, ld] (grb_hstu_bias_index_jagged)."""

    def __init__(self, pad_u8: torch.Tensor, timestamps: Optional[torch.Tensor], pos_bucket: Optional[torch.Tensor],
                 time_thr: torch.Tensor, num_time_buckets: int = 64, num_pos_buckets: int = 32, pos_uniform=None,
                 may_defer: bool = True, offsets: Optional[torch.Tensor] = None, max_len: Optional[int] = None):
        # may_defer=False builds the index on the caller's stream even under the deferred schedule (the custom ops, whose
        # callers order and free everything by that stream); pos_bucket may be None when pos_uniform is given
        require_cuda(pad_u8, offsets)
        self.offsets = offsets
        if offsets is None:
            B, L = pad_u8.shape
            self.T = B * L
        else:
            B, L = offsets.numel() - 1, int(max_len)
            self.T = pad_u8.numel()
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
        self._build_bias_index(may_defer)

    def _build_bias_index(self, may_defer: bool):
        B, L, dev = self.B, self.L, self.pad.device
        rows = (B, L) if self.offsets is None else (self.T,)
        self.bias_index = torch.empty(*rows, self.ld, dtype=torch.int16, device=dev)
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
        if self.offsets is None:
            call(dev, "grb_hstu_bias_index", ptr(self.timestamps), ptr(self.pad), ptr(self.time_thr), ptr(pb_arg), B, L, npos_arg, nt,
                 ptr(self.bias_index), self.ld)
        else:
            call(dev, "grb_hstu_bias_index_jagged", ptr(self.timestamps), ptr(self.pad), ptr(self.offsets), ptr(self.time_thr), ptr(pb_arg),
                 B, self.T, L, npos_arg, nt, ptr(self.bias_index), self.ld)

    def struct(self) -> HstuSeq:
        return HstuSeq(ptr(self.bias_index), self.ld, 1 if self.timestamps is not None else 0, 1 if self.pos_uniform else 0,
                       self.pos_bucket0)


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
    return _lib.host_bytes("grb_hstu_layer_saved_bytes", C.byref(dims))


def hstu_block_forward(dims: HstuDims, params, bf16w: dict, has_time: bool, meta: SeqMeta, x: torch.Tensor):
    """One HSTU block (grb_hstu_layer_forward): x [B, L, D] fp32 contiguous -> (y, saved-for-backward blob).  A packed ``meta``
    (offsets set) takes x [T, D] and runs grb_hstu_layer_forward_jagged."""
    if meta.offsets is None:
        saved = workspace(x.device, "grb_hstu_layer_saved_bytes", C.byref(dims))
    else:
        saved = workspace(x.device, "grb_hstu_layer_saved_bytes_jagged", C.byref(dims), meta.T)
    y = torch.empty_like(x)
    pstruct, seq = _layer_param_struct(params, bf16w, has_time), meta.struct()
    if meta.offsets is None:
        call(x.device, "grb_hstu_layer_forward", C.byref(dims), C.byref(pstruct), C.byref(seq), ptr(x), ptr(y), ptr(saved))
    else:
        call(x.device, "grb_hstu_layer_forward_jagged", C.byref(dims), C.byref(pstruct), C.byref(seq), ptr(meta.offsets), meta.T, ptr(x),
             ptr(y), ptr(saved))
    return y, saved


def hstu_block_backward(dims: HstuDims, params, bf16w: dict, has_time: bool, meta: SeqMeta, dy: torch.Tensor, saved: torch.Tensor,
                        sink: Optional[dict] = None):
    """grb_hstu_layer_backward -> (dx, parameter gradients in PARAM_ORDER, None where a parameter is absent).  With a ``sink``
    (name -> view of the flat gradient buffer of genrec_b200.optim.FlatAdam) the gradients accumulate there, and the weight
    gradients follow the deferred schedule when it is on."""
    if sink is not None:
        grads = [sink[n] if q is not None else None for n, q in zip(PARAM_ORDER, params)]
    else:
        grads = [torch.zeros(q.shape, dtype=torch.float32, device=dy.device) if q is not None else None for q in params]
    pstruct, gstruct, seq = _layer_param_struct(params, bf16w, has_time), HstuLayerGrads(*[ptr(g) for g in grads]), meta.struct()
    dyc = dy.contiguous().float()
    dx = torch.empty_like(dyc)
    if meta.offsets is None:
        ws = workspace(dy.device, "grb_hstu_layer_workspace_bytes", C.byref(dims))
    else:
        ws = workspace(dy.device, "grb_hstu_layer_workspace_bytes_jagged", C.byref(dims), meta.T)
    deferred = _defer_for_call(_DEFER["on"] and sink is not None)
    if meta.offsets is None:
        call(dy.device, "grb_hstu_layer_backward", C.byref(dims), C.byref(pstruct), C.byref(seq), ptr(dyc), ptr(saved), ptr(dx),
             C.byref(gstruct), ptr(ws))
    else:
        call(dy.device, "grb_hstu_layer_backward_jagged", C.byref(dims), C.byref(pstruct), C.byref(seq), ptr(meta.offsets), meta.T,
             ptr(dyc), ptr(saved), ptr(dx), C.byref(gstruct), ptr(ws))
    if deferred:
        _DEFER["keep"].append((ws, saved, dyc))     # still read by the deferred dW GEMM
    return dx, grads


class HstuLayerFn(torch.autograd.Function):
    """One HSTU block.  forward = grb_hstu_layer_forward, backward = grb_hstu_layer_backward; on a packed ``meta`` (x [T, D]) their
    _jagged forms, with B = the sequence count and L = max_len."""

    @staticmethod
    def forward(ctx, x, meta: SeqMeta, cfg: dict, bf16w: dict, *params):
        # params in PARAM_ORDER (fp32 masters; time_table may be None)
        require_cuda(x)
        if meta.offsets is None:
            B, L, D = x.shape
        else:
            B, L, D = meta.B, meta.L, x.shape[-1]
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


def check_jagged_batch(what: str, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int, max_len_limit: int) -> torch.Tensor:
    """Argument check of a packed batch before any launch (HSTU and SASRec) -> offsets on input_ids' device.  input_ids must be a
    non-empty [T] int64 tensor, offsets a [B+1] int64 tensor with 1 <= B <= 65535 (the attention grid's z dimension), max_len an int
    in [1, max_len_limit].  CPU offsets are refused with ValueError unless offsets[0] == 0, they never decrease, no length exceeds
    max_len and offsets[B] <= T; device offsets are not read on the host (CUDA graphs), and the kernels keep a malformed one inside
    the T rows."""
    if input_ids.dim() != 1 or input_ids.numel() == 0 or input_ids.dtype != torch.int64:
        raise ValueError(f"{what}: input_ids must be a non-empty [T] int64 tensor, got {tuple(input_ids.shape)} {input_ids.dtype}")
    T = input_ids.numel()
    if not isinstance(offsets, torch.Tensor) or offsets.dim() != 1 or offsets.numel() < 2 or offsets.dtype != torch.int64:
        raise ValueError(f"{what}: offsets must be a [B+1] int64 tensor with B >= 1")
    if offsets.numel() - 1 > 65535:
        raise ValueError(f"{what}: B = {offsets.numel() - 1} sequences exceeds 65535 (the attention grid's z dimension)")
    if isinstance(max_len, bool) or not isinstance(max_len, int) or not 1 <= max_len <= max_len_limit:
        raise ValueError(f"{what}: max_len must be an int in [1, {max_len_limit}], got {max_len!r}")
    if not offsets.is_cuda:
        o = offsets
        if int(o[0]) != 0:
            raise ValueError(f"{what}: offsets[0] must be 0, got {int(o[0])}")
        lens = o[1:] - o[:-1]
        if bool((lens < 0).any()):
            raise ValueError(f"{what}: offsets must be non-decreasing")
        if int(lens.max()) > max_len:
            raise ValueError(f"{what}: a sequence of length {int(lens.max())} exceeds max_len {max_len}")
        if int(o[-1]) > T:
            raise ValueError(f"{what}: offsets[B] = {int(o[-1])} exceeds the {T} token rows")
    elif offsets.device != input_ids.device:
        raise ValueError(f"{what}: offsets must be on the CPU or on {input_ids.device}, got {offsets.device}")
    require_cuda(input_ids)
    ensure_device(input_ids.device)
    return offsets.to(input_ids.device)


def last_rows_jagged(x: torch.Tensor, offsets: torch.Tensor) -> torch.Tensor:
    """x [T, D] of a packed batch -> [B, D]: the last row of each sequence, offsets[b+1] - 1, and zeros for a sequence of length 0."""
    last = (offsets[1:] - 1).clamp(0, x.shape[0] - 1)
    return torch.where((offsets[1:] > offsets[:-1])[:, None], x.index_select(0, last), torch.zeros((), dtype=x.dtype, device=x.device))


class EmbedFn(torch.autograd.Function):
    """x = dropout(E[ids] * scale (+ pos)) ; also emits the uint8 pad flags.  With ``offsets`` ([B+1] int64 on the device) and
    ``max_len`` the batch is packed (ids [T] -> x [T, D], pad [T]) and each token takes SASRec's position row P - n_b + i, P the
    longest sequence, derived on the device (grb_embed_forward_jagged); rows outside every sequence get x = 0 and pad = 1."""

    @staticmethod
    def forward(ctx, ids, table, pos_table, scale, mask_pad_rows, p, seed, seed_dev, sink=None, offsets=None, max_len=None):
        require_cuda(ids, table)
        require_i64(ids)
        require_f32(table, pos_table)
        ctx.sink = sink
        ctx.jagged = None
        D = table.shape[1]
        ids = ids.contiguous()
        if offsets is not None:
            T = ids.numel()
            B = offsets.numel() - 1
            x = torch.empty(T, D, dtype=torch.float32, device=ids.device)
            pad = torch.empty(T, dtype=torch.uint8, device=ids.device)
            positions = torch.empty(T, dtype=torch.int32, device=ids.device)
            call(ids.device, "grb_embed_forward_jagged", ptr(ids), ptr(table.detach()), ptr(pos_table.detach()), ptr(offsets), B, T,
                 int(max_len), D, float(scale), int(mask_pad_rows), float(p), int(seed), ptr(seed_dev), ptr(x), ptr(pad), ptr(positions))
            ids = torch.where(positions >= 0, ids, 0)   # the idle rows' x does not depend on the table
            ctx.jagged = (offsets, B, T, int(max_len))
        else:
            B, L = ids.shape
            x = torch.empty(B, L, D, dtype=torch.float32, device=ids.device)
            pad = torch.empty(B, L, dtype=torch.uint8, device=ids.device)
            call(ids.device, "grb_embed_forward", ptr(ids), ptr(table.detach()),
                 ptr(pos_table.detach()) if pos_table is not None else None, ptr(x), ptr(pad), B, L, D, float(scale), int(mask_pad_rows),
                 float(p), int(seed), ptr(seed_dev))
        ctx.save_for_backward(ids)
        ctx.args = (table.shape, None if pos_table is None else pos_table.shape, scale, mask_pad_rows, p, seed, seed_dev)
        ctx.mark_non_differentiable(pad)
        return x, pad

    @staticmethod
    def backward(ctx, dx, _dpad):
        (ids,) = ctx.saved_tensors
        tshape, pshape, scale, mask_pad_rows, p, seed, seed_dev = ctx.args
        D = tshape[1]
        dx = dx.contiguous().float()
        if ctx.sink is not None:
            dtable, dpos = ctx.sink
        else:
            dtable = torch.zeros(tshape, dtype=torch.float32, device=dx.device)
            dpos = torch.zeros(pshape, dtype=torch.float32, device=dx.device) if pshape is not None else None
        order = torch.sort(ids.reshape(-1), stable=True).indices   # tokens grouped by id, in token order
        scratch = torch.empty(ids.numel(), D, dtype=torch.float32, device=dx.device)
        if ctx.jagged is not None:
            offsets, B, T, max_len = ctx.jagged
            call(dx.device, "grb_embed_backward_jagged", ptr(ids), ptr(order), ptr(dx), ptr(dtable), ptr(dpos), ptr(offsets), B, T, max_len,
                 D, float(scale), int(mask_pad_rows), float(p), int(seed), ptr(seed_dev), ptr(scratch))
        else:
            B, L = ids.shape
            call(dx.device, "grb_embed_backward", ptr(ids), ptr(order), ptr(dx), ptr(dtable), ptr(dpos), B, L, D, float(scale),
                 int(mask_pad_rows), float(p), int(seed), ptr(seed_dev), ptr(scratch))
        if ctx.sink is not None:
            return (None,) * 11
        return None, dtable, dpos, None, None, None, None, None, None, None, None


def _head_grad_buffers(ctx, xc, ln_g, ln_b, table, sink, unit_loss_grad):
    """-> (dx, dg, db, dtable, direct) for a loss head's forward: the sink's views when the kernels may add straight into it
    (``direct``), fresh zeroed tensors when gradients are needed otherwise, ``None``s for a loss-only call."""
    need_grad = any(ctx.needs_input_grad[:4])
    direct = need_grad and sink is not None and unit_loss_grad
    ctx.sink, ctx.direct = sink, direct
    if direct:
        return (torch.empty_like(xc), *sink, True)
    if not need_grad:
        return None, None, None, None, False
    return (torch.empty_like(xc), torch.zeros_like(ln_g, dtype=torch.float32), torch.zeros_like(ln_b, dtype=torch.float32),
            torch.zeros(table.shape, dtype=torch.float32, device=xc.device), False)


def _head_loss_backward(ctx, dloss, n_inputs):
    """backward of both loss heads: ``ctx.grads`` scaled by ``dloss`` (see ``HeadLossFn``), ``None`` for the other inputs."""
    dx, dg, db, dtable = ctx.grads
    ctx.grads = None
    if dx is None:
        return (None,) * n_inputs
    if ctx.direct:
        call(dx.device, "grb_assert_unit_scalar", ptr(dloss.detach().float().contiguous()))
        return (dx,) + (None,) * (n_inputs - 1)
    if ctx.sink is not None:
        sg, sb, st = ctx.sink
        sg.add_(dg * dloss); sb.add_(db * dloss); st.addcmul_(dtable, dloss)
        return (dx * dloss,) + (None,) * (n_inputs - 1)
    return (dx * dloss, dg * dloss, db * dloss, dtable * dloss) + (None,) * (n_inputs - 4)


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
        require_cuda(x, table, targets)
        require_i64(targets)
        require_f32(ln_g, ln_b, table)
        B, L, D = x.shape
        T, Cn = B * L, table.shape[0]
        xc = x.detach().contiguous().float()
        tg = targets.contiguous()
        dx, dg, db, dtable, direct = _head_grad_buffers(ctx, xc, ln_g, ln_b, table, sink, unit_loss_grad)
        loss = torch.empty((), dtype=torch.float32, device=x.device)   # zeroed on the device by the target-count kernel
        ws = workspace(x.device, "grb_head_workspace_bytes", T, D, Cn)
        deferred = _defer_for_call(_DEFER["on"] and direct)
        call(x.device, "grb_head_loss_forward_backward", ptr(xc), ptr(ln_g.detach()), ptr(ln_b.detach()), float(eps), ptr(table_bf16),
             ptr(tg), T, D, Cn, ptr(loss), ptr(dx), ptr(dtable), ptr(dg), ptr(db), ptr(ws))
        if deferred:
            _DEFER["keep"].append((ws, xc, tg))                   # xf, the shifts and the targets are still read by the deferred dE pass
        ctx.grads = (dx, dg, db, dtable)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        return _head_loss_backward(ctx, dloss, 9)


def head_sampled_loss_raw(x, ln_g, ln_b, table_bf16, targets, negatives, log_q, eps, grads=None):
    """grb_head_sampled_loss_forward_backward on x [T, D]: -> loss (0-dim fp32).  ``grads = (dx, dtable, dln_g, dln_b)``: dx is
    written, the other three are accumulated into; ``None``: loss only."""
    require_cuda(x, table_bf16, targets, negatives, log_q)
    require_i64(targets, negatives)
    require_f32(x, ln_g, ln_b, log_q)
    T, D = x.shape
    Cn, N = table_bf16.shape[0], negatives.numel()
    if negatives.dim() != 1:
        raise _lib.GrbError(f"genrec_b200 error -1: negatives must be one [N] vector shared by every token (got shape {tuple(negatives.shape)})")
    if log_q is not None and tuple(log_q.shape) != (Cn,):
        raise _lib.GrbError(f"genrec_b200 error -1: log_q must be [{Cn}] (one entry per table row), got {tuple(log_q.shape)}")
    for t in (negatives, log_q):
        if t is not None and t.device != x.device:
            raise _lib.GrbError(f"genrec_b200 error -1: negatives / log_q must live on the model's device {x.device} (got {t.device})")
    neg = negatives.contiguous()
    lq = log_q.detach().contiguous() if log_q is not None else None
    loss = torch.empty((), dtype=torch.float32, device=x.device)   # zeroed on the device by the target-count kernel
    ws = workspace(x.device, "grb_head_sampled_workspace_bytes", T, D, N)
    dx, dtable, dg, db = grads if grads is not None else (None,) * 4
    call(x.device, "grb_head_sampled_loss_forward_backward", ptr(x), ptr(ln_g.detach()), ptr(ln_b.detach()), float(eps), ptr(table_bf16),
         ptr(targets), ptr(neg), ptr(lq), T, D, Cn, N, ptr(loss), ptr(dx), ptr(dtable), ptr(dg), ptr(db), ptr(ws))
    return loss


class SampledHeadLossFn(torch.autograd.Function):
    """loss = sampled softmax of LN(x) against E[targets] and the shared ``negatives`` [N], scores corrected by ``-log_q`` (see
    grb_head_sampled_loss_forward_backward).  ``sink`` / ``unit_loss_grad`` behave as in ``HeadLossFn``."""

    @staticmethod
    def forward(ctx, x, ln_g, ln_b, table, table_bf16, targets, negatives, log_q, eps, sink=None, unit_loss_grad=False):
        require_f32(table)
        B, L, D = x.shape
        xc = x.detach().contiguous().float()
        tg = targets.contiguous().view(-1)
        dx, dg, db, dtable, _ = _head_grad_buffers(ctx, xc, ln_g, ln_b, table, sink, unit_loss_grad)
        loss = head_sampled_loss_raw(xc.view(B * L, D), ln_g, ln_b, table_bf16, tg, negatives, log_q, eps,
                                     (dx.view(B * L, D), dtable, dg, db) if dx is not None else None)
        ctx.grads = (dx, dg, db, dtable)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        return _head_loss_backward(ctx, dloss, 11)


def head_logits(x, ln_g, ln_b, table, table_bf16, eps) -> torch.Tensor:
    """fp32 logits [B, L, C] (no autograd - inference / API parity path)."""
    require_cuda(x, table)
    B, L, D = x.shape
    T, Cn = B * L, table.shape[0]
    xc = x.detach().contiguous().float()
    logits = torch.empty(B, L, Cn, dtype=torch.float32, device=x.device)
    ws = workspace(x.device, "grb_head_workspace_bytes", T, D, Cn)
    call(x.device, "grb_head_logits", ptr(xc), ptr(ln_g.detach()), ptr(ln_b.detach()), float(eps), ptr(table_bf16), T, D, Cn, ptr(logits),
         ptr(ws))
    return logits


class TopItems(NamedTuple):
    """The k best items per row, best first: ``scores`` [R, k] fp32 and ``items`` [R, k] int64 (slots without an eligible item hold
    score -inf and item 0)."""
    scores: torch.Tensor
    items: torch.Tensor


TOPK_MAX_K, TOPK_MAX_EXCLUDE = 64, 16384


def check_topk_args(k: int, exclude: Optional[torch.Tensor], rows: int, device) -> None:
    """ValueError unless 1 <= k <= 64 and ``exclude`` is None or an int64 [rows, E <= 16384] tensor on ``device``."""
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= TOPK_MAX_K:
        raise ValueError(f"top_k must be an int in [1, {TOPK_MAX_K}], got {k!r}")
    check_exclude_arg(exclude, rows, device)


def check_exclude_arg(exclude: Optional[torch.Tensor], rows: int, device) -> None:
    """ValueError unless ``exclude`` is None or an int64 [rows, E <= 16384] tensor on ``device``."""
    if exclude is None:
        return
    if not isinstance(exclude, torch.Tensor) or exclude.dim() != 2 or exclude.shape[0] != rows:
        raise ValueError(f"exclude must be a [{rows}, E] tensor (one row per input row), got "
                         f"{tuple(exclude.shape) if isinstance(exclude, torch.Tensor) else type(exclude).__name__}")
    if exclude.dtype != torch.int64:
        raise ValueError(f"exclude must be int64, got {exclude.dtype}")
    if exclude.device != torch.device(device):
        raise ValueError(f"exclude must be on {device}, got {exclude.device}")
    if exclude.shape[1] > TOPK_MAX_EXCLUDE:
        raise ValueError(f"exclude holds at most {TOPK_MAX_EXCLUDE} ids per row, got {exclude.shape[1]}")


def _sweep_inputs(x, table_bf16, exclude, check_rows, query, *k):
    """What head_topk and head_rank_metrics share: x must be [R, D], and ``check_rows(R)`` runs the head's own argument checks.
    -> (x as contiguous fp32, exclude or None when it holds no ids, E, the workspace of size query ``query(R, D, C, *k, E)``)"""
    if x.dim() != 2:
        raise ValueError(f"x must be [R, D], got {tuple(x.shape)}")
    R, D = x.shape
    check_rows(R)
    ex = exclude.contiguous() if exclude is not None and exclude.shape[1] > 0 else None
    E = ex.shape[1] if ex is not None else 0
    return x.detach().contiguous().float(), ex, E, workspace(x.device, query, R, D, table_bf16.shape[0], *k, E)


def head_topk(x, ln_g, ln_b, table_bf16, eps, k: int, exclude: Optional[torch.Tensor] = None) -> TopItems:
    """The ``k`` best items of every row of ``x`` [R, D] under the tied head, without forming the logits (grb_head_topk): scores are
    bit-identical to ``head_logits`` of the same rows; item 0 and the row's ``exclude`` ids ([R, E] int64, any order) never appear;
    ties go to the lower item id.  Inference only (no autograd)."""
    require_cuda(x, table_bf16)
    xc, ex, E, ws = _sweep_inputs(x, table_bf16, exclude, lambda R: check_topk_args(k, exclude, R, x.device),
                                  "grb_head_topk_workspace_bytes", k)
    R, D = x.shape
    Cn = table_bf16.shape[0]
    scores = torch.empty(R, k, dtype=torch.float32, device=x.device)
    items = torch.empty(R, k, dtype=torch.int64, device=x.device)
    call(x.device, "grb_head_topk", ptr(xc), ptr(ln_g.detach()), ptr(ln_b.detach()), float(eps), ptr(table_bf16), R, D, Cn, k, ptr(ex), E,
         ptr(scores), ptr(items), ptr(ws))
    return TopItems(scores, items)


CANDIDATES_MAX_K = 2048


def check_candidates_args(k: int, exclude: Optional[torch.Tensor], rows: int, device) -> None:
    """ValueError unless 1 <= k <= 2048 and ``exclude`` is None or an int64 [rows, E <= 16384] tensor on ``device``."""
    if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= CANDIDATES_MAX_K:
        raise ValueError(f"num_candidates must be an int in [1, {CANDIDATES_MAX_K}], got {k!r}")
    check_exclude_arg(exclude, rows, device)


def head_candidates(x, ln_g, ln_b, table_bf16, eps, k: int, exclude: Optional[torch.Tensor] = None) -> TopItems:
    """``head_topk`` for up to 2048 items per row (grb_head_candidates): the ``k`` best items of every row of ``x`` [R, D] under
    the tied head, best first, without forming the logits.  Same rules: scores bit-identical to ``head_logits``, item 0 and the
    row's ``exclude`` ids never appear, ties go to the lower item id, (-inf, 0) where no eligible item is left.  Memory grows with
    R * k and R * E, not with the catalog.  Inference only (no autograd)."""
    require_cuda(x, table_bf16)
    xc, ex, E, ws = _sweep_inputs(x, table_bf16, exclude, lambda R: check_candidates_args(k, exclude, R, x.device),
                                  "grb_head_candidates_workspace_bytes", k)
    R, D = x.shape
    Cn = table_bf16.shape[0]
    scores = torch.empty(R, k, dtype=torch.float32, device=x.device)
    items = torch.empty(R, k, dtype=torch.int64, device=x.device)
    call(x.device, "grb_head_candidates", ptr(xc), ptr(ln_g.detach()), ptr(ln_b.detach()), float(eps), ptr(table_bf16), R, D, Cn, k,
         ptr(ex), E, ptr(scores), ptr(items), ptr(ws))
    return TopItems(scores, items)


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
    call(lg.device, "grb_eval_rank_metrics", ptr(lg), ptr(targets.contiguous()), B, Cn, ptr(metrics), ptr(ranks))
    return (metrics, ranks) if want_ranks else metrics


def head_rank_metrics(x, ln_g, ln_b, table_bf16, eps, targets: torch.Tensor, metrics: Optional[torch.Tensor] = None,
                      exclude: Optional[torch.Tensor] = None, want_ranks: bool = False):
    """``eval_rank_metrics(head_logits(x))`` without the [R, C] logits (grb_head_rank): x [R, D] fp32, targets [R] int64 ->
    metrics [6] fp32 accumulated on the device (Recall@{1,5,10} hit counts, NDCG@{1,5,10} sums), and with ``want_ranks`` the
    int32 ranks [R] too.  The target's rank is counted while the head scores the table, with scores bit-identical to
    ``head_logits``, so the ranks equal ``eval_rank_metrics``' exactly.  ``exclude`` ([R, E] int64, any order, E <= 16384) removes
    ids from the count; a row whose target is 0, out of 1..C-1 or excluded gets rank 0 and adds nothing.  Memory grows with R and
    R * E, not with the catalog.  Inference only (no autograd)."""
    require_cuda(x, table_bf16, targets)
    require_i64(targets)

    def check_rows(R):
        if targets.shape != (R,):
            raise ValueError(f"targets must be [{R}] (one per row of x), got {tuple(targets.shape)}")
        check_exclude_arg(exclude, R, x.device)

    xc, ex, E, ws = _sweep_inputs(x, table_bf16, exclude, check_rows, "grb_head_rank_workspace_bytes")
    R, D = x.shape
    Cn = table_bf16.shape[0]
    if metrics is None:
        metrics = torch.zeros(6, dtype=torch.float32, device=x.device)
    ranks = torch.empty(R, dtype=torch.int32, device=x.device) if want_ranks else None
    call(x.device, "grb_head_rank", ptr(xc), ptr(ln_g.detach()), ptr(ln_b.detach()), float(eps), ptr(table_bf16), R, D, Cn,
         ptr(targets.contiguous()), ptr(ex), E, ptr(metrics), ptr(ranks), ptr(ws))
    return (metrics, ranks) if want_ranks else metrics


# ------------------------------------------------------------------------------------------------ attention core alone
def hstu_attention_fwd(P: torch.Tensor, meta: SeqMeta, H: int, pos_table: torch.Tensor, time_table: Optional[torch.Tensor],
                       ntime: int = 64) -> torch.Tensor:
    """P [B, L, 4D] bf16 = silu(x Wp^T + b) = [U | V | Q | K]  ->  O [B, L, D] bf16 (hstu.py:244-267)."""
    require_cuda(P)
    B, L, D4 = P.shape
    D = D4 // 4
    has_time = time_table is not None and meta.timestamps is not None
    dims = _dims(B, L, D, H, pos_table.shape[0], ntime if has_time else 0, 0.0, 0, None, 0)
    O = torch.empty(B, L, D, dtype=torch.bfloat16, device=P.device)
    seq = meta.struct()
    call(P.device, "grb_hstu_attention_forward", C.byref(dims), ptr(pos_table), ptr(time_table) if has_time else None, C.byref(seq),
         ptr(P), ptr(O))
    return O


def hstu_attention_bwd(P, zp, dO, meta: SeqMeta, H: int, pos_table, time_table, ntime: int = 64):
    """-> dzp [B, L, 4D] bf16 (columns V, Q, K written; U untouched = 0), dpos_table, dtime_table (fp32)."""
    B, L, D4 = P.shape
    D = D4 // 4
    has_time = time_table is not None and meta.timestamps is not None
    dims = _dims(B, L, D, H, pos_table.shape[0], ntime if has_time else 0, 0.0, 0, None, 0)
    dzp = torch.zeros(B, L, D4, dtype=torch.bfloat16, device=P.device)
    dpos = torch.zeros_like(pos_table, dtype=torch.float32)
    dtime = torch.zeros_like(time_table, dtype=torch.float32) if has_time else None
    scratch = workspace(P.device, "grb_hstu_attention_scratch_bytes", C.byref(dims))
    seq = meta.struct()
    call(P.device, "grb_hstu_attention_backward", C.byref(dims), ptr(pos_table), ptr(time_table) if has_time else None, C.byref(seq),
         ptr(P), ptr(zp), ptr(dO), ptr(dzp), ptr(dpos), ptr(dtime), ptr(scratch))
    return dzp, dpos, dtime


# ------------------------------------------------------------------------------------------------ cached incremental inference
def hstu_cache_append(cache: _lib.HstuCache, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor],
                      offsets: Optional[torch.Tensor] = None, max_len: Optional[int] = None):
    """input_ids / timestamps [B, n] int64 -> (positions [B, n] int32, last_row [B] int32); advances the cache's lengths and stores
    the chunk's timestamps (grb_hstu_cache_append).  With ``offsets`` ([B+1] int64 on the device) and ``max_len`` the chunk is
    packed: input_ids / timestamps [T] -> positions [T], last_row [B] holding token rows (grb_hstu_cache_append_jagged)."""
    require_cuda(input_ids, timestamps, offsets)
    require_i64(input_ids, timestamps, offsets)
    dev = input_ids.device
    ids = input_ids.contiguous()
    ts = timestamps.contiguous() if timestamps is not None else None
    if offsets is not None:
        B, T = offsets.numel() - 1, ids.numel()
        positions = torch.empty(T, dtype=torch.int32, device=dev)
        last_row = torch.empty(B, dtype=torch.int32, device=dev)
        call(dev, "grb_hstu_cache_append_jagged", C.byref(cache), ptr(ids), ptr(ts), ptr(offsets.contiguous()), B, T, int(max_len),
             ptr(positions), ptr(last_row))
        return positions, last_row
    B, n = input_ids.shape
    positions = torch.empty(B, n, dtype=torch.int32, device=dev)
    last_row = torch.empty(B, dtype=torch.int32, device=dev)
    call(dev, "grb_hstu_cache_append", C.byref(cache), ptr(ids), ptr(ts), n, ptr(positions), ptr(last_row))
    return positions, last_row


def hstu_layer_extend(x: torch.Tensor, cache, layer: int, positions: torch.Tensor, pos_bucket: Optional[torch.Tensor],
                      pos_bucket0: int, time_thr: torch.Tensor, H: int, npos: int, ntime: int, bf16w: dict, params,
                      users: Optional[torch.Tensor] = None, offsets: Optional[torch.Tensor] = None,
                      max_len: Optional[int] = None) -> torch.Tensor:
    """One block on a chunk against the cache: x [B, n, D] fp32 -> y [B, n, D] fp32.  ``cache`` is a dense ``HstuCache``
    (grb_hstu_layer_extend) or an ``HstuPool`` with ``users`` [B] int64 on the device (grb_hstu_layer_extend_paged).  ``params`` in
    PARAM_ORDER (time_table None or ntime = 0: no temporal term), ``bf16w`` the three bf16 weight mirrors.  With ``offsets``
    ([B+1] int64 on the device) and ``max_len`` the chunk is packed: x [T, D] -> y [T, D] (the ``_jagged`` entry points)."""
    require_cuda(x)
    require_f32(x)
    xc = x.contiguous()
    D = x.shape[-1]
    if offsets is not None:
        B, n, T = offsets.numel() - 1, int(max_len), x.numel() // D
    else:
        B, n, D = x.shape
    has_time = params[PARAM_ORDER.index("time_table")] is not None and ntime > 0
    dims = _dims(B, n, D, H, npos, ntime if has_time else 0, 0.0, 0, None, layer)
    pstruct = _layer_param_struct(params, bf16w, has_time)
    paged = isinstance(cache, _lib.HstuPool)
    dev = x.device
    if offsets is not None and paged:
        ws = workspace(dev, "grb_hstu_layer_extend_paged_workspace_bytes_jagged", C.byref(dims), C.byref(cache), T)
    elif offsets is not None:
        ws = workspace(dev, "grb_hstu_layer_extend_workspace_bytes_jagged", C.byref(dims), cache.capacity, T)
    elif paged:
        ws = workspace(dev, "grb_hstu_layer_extend_paged_workspace_bytes", C.byref(dims), C.byref(cache))
    else:
        ws = workspace(dev, "grb_hstu_layer_extend_workspace_bytes", C.byref(dims), cache.capacity)
    y = torch.empty_like(xc)
    head = (C.byref(dims), C.byref(pstruct), C.byref(cache), layer)
    tail = (ptr(positions), ptr(pos_bucket), int(pos_bucket0), ptr(time_thr), ptr(xc), ptr(y), ptr(ws))
    if offsets is not None and paged:
        call(dev, "grb_hstu_layer_extend_paged_jagged", *head, ptr(users), ptr(offsets), T, *tail)
    elif offsets is not None:
        call(dev, "grb_hstu_layer_extend_jagged", *head, ptr(offsets), T, *tail)
    elif paged:
        call(dev, "grb_hstu_layer_extend_paged", *head, ptr(users), *tail)
    else:
        call(dev, "grb_hstu_layer_extend", *head, *tail)
    return y


def hstu_pool_append(pool: _lib.HstuPool, users: torch.Tensor, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor],
                     offsets: Optional[torch.Tensor] = None, max_len: Optional[int] = None):
    """users [B] int64 and input_ids / timestamps [B, n] int64 on the device -> (positions [B, n] int32, last_row [B] int32, room [B]
    int32); hands out the pages the chunk needs and stores its timestamps (grb_hstu_pool_append).  With ``offsets`` ([B+1] int64 on
    the device) and ``max_len`` the chunk is packed: input_ids / timestamps [T] -> positions [T], last_row [B] holding token rows
    (grb_hstu_pool_append_jagged)."""
    require_cuda(users, input_ids, timestamps, offsets)
    require_i64(users, input_ids, timestamps, offsets)
    dev = input_ids.device
    B = users.numel() if offsets is not None else input_ids.shape[0]
    ids = input_ids.contiguous()
    ts = timestamps.contiguous() if timestamps is not None else None
    positions = torch.empty(ids.shape, dtype=torch.int32, device=dev)
    last_row = torch.empty(B, dtype=torch.int32, device=dev)
    room = torch.empty(B, dtype=torch.int32, device=dev)
    if offsets is not None:
        call(dev, "grb_hstu_pool_append_jagged", C.byref(pool), ptr(users.contiguous()), B, ptr(ids), ptr(ts), ptr(offsets.contiguous()),
             ids.numel(), int(max_len), ptr(positions), ptr(last_row), ptr(room))
    else:
        call(dev, "grb_hstu_pool_append", C.byref(pool), ptr(users.contiguous()), B, ptr(ids), ptr(ts), ids.shape[1], ptr(positions),
             ptr(last_row), ptr(room))
    return positions, last_row, room


def hstu_pool_release(pool: _lib.HstuPool, users: torch.Tensor, last_hidden: Optional[torch.Tensor]) -> None:
    """Return the pages of users [B] int64 (device) to the pool and zero their lengths, flags and rows of last_hidden [*, D] fp32."""
    require_cuda(users, last_hidden)
    require_i64(users)
    D = last_hidden.shape[1] if last_hidden is not None else 0
    call(users.device, "grb_hstu_pool_release", C.byref(pool), ptr(users.contiguous()), users.numel(), ptr(last_hidden), D)


# ------------------------------------------------------------------------------------------------ SASRec, TIGER and COBRA pieces
def layernorm_fwd(x, g, b, eps, want_bf16=True, want_f32=False):
    T, D = x.numel() // x.shape[-1], x.shape[-1]
    yb = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device) if want_bf16 else None
    yf = torch.empty(x.shape, dtype=torch.float32, device=x.device) if want_f32 else None
    st = torch.empty(T, 2, dtype=torch.float32, device=x.device)
    call(x.device, "grb_layernorm_forward", ptr(x), ptr(g), ptr(b), float(eps), T, D, ptr(yb), ptr(yf), ptr(st))
    return yb, yf, st


def layernorm_bwd(dy, x, st, g, residual=None):
    T, D = x.numel() // x.shape[-1], x.shape[-1]
    dx = torch.empty_like(x)
    dg = torch.zeros_like(g)
    db = torch.zeros_like(g)
    ws = workspace(x.device, "grb_layernorm_backward_workspace_bytes", T, D)
    call(x.device, "grb_layernorm_backward", ptr(dy), ptr(x), ptr(st), ptr(g), ptr(residual), T, D, ptr(dx), ptr(dg), ptr(db), ptr(ws))
    return dx, dg, db


def rmsnorm_fwd(x, w, eps, want_bf16=True, want_f32=False):
    """T5 RMS norm of x [..., D] fp32 contiguous -> (y bf16 | None, y fp32 | None, rstd fp32 [T])"""
    T, D = x.numel() // x.shape[-1], x.shape[-1]
    yb = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device) if want_bf16 else None
    yf = torch.empty(x.shape, dtype=torch.float32, device=x.device) if want_f32 else None
    rstd = torch.empty(T, dtype=torch.float32, device=x.device)
    call(x.device, "grb_rmsnorm_forward", ptr(x), ptr(w), float(eps), T, D, ptr(yb), ptr(yf), ptr(rstd))
    return yb, yf, rstd


def rmsnorm_bwd(dy, x, rstd, w, residual=None):
    """-> (dx fp32 (+ residual), dw fp32), dw summed in a fixed order"""
    T, D = x.numel() // x.shape[-1], x.shape[-1]
    dx = torch.empty_like(x)
    dw = torch.zeros_like(w)
    ws = workspace(x.device, "grb_rmsnorm_backward_workspace_bytes", T, D)
    call(x.device, "grb_rmsnorm_backward", ptr(dy), ptr(x), ptr(rstd), ptr(w), ptr(residual), T, D, ptr(dx), ptr(dw), ptr(ws))
    return dx, dw


def linear_fwd(xb, wb, bias, act, p=0.0, seed=0, seed_dev=None, site=0, out=None):
    """z = xb @ wb^T + bias (bf16) ; act: 0 none, 1 silu, 2 relu -> returns (z, act(z) with dropout); out: a contiguous bf16 tensor of
    z's shape that receives z"""
    T, K = xb.numel() // xb.shape[-1], xb.shape[-1]
    N = wb.shape[0]
    z = torch.empty(*xb.shape[:-1], N, dtype=torch.bfloat16, device=xb.device) if out is None else out
    a = torch.empty_like(z) if act else None
    call(xb.device, "grb_linear_forward", ptr(xb), ptr(wb), ptr(bias), T, N, K, act, ptr(z), ptr(a), float(p), int(seed), ptr(seed_dev),
         site)
    return z, a


def linear_residual_fwd(xb, wb, bias, residual, row_scale=None, p=0.0, seed=0, seed_dev=None, site=0):
    T, K = xb.numel() // xb.shape[-1], xb.shape[-1]
    N = wb.shape[0]
    y = torch.empty(*xb.shape[:-1], N, dtype=torch.float32, device=xb.device)
    call(xb.device, "grb_linear_residual_forward", ptr(xb), ptr(wb), ptr(bias), ptr(residual), ptr(row_scale), T, N, K, ptr(y), float(p),
         int(seed), ptr(seed_dev), site)
    return y


def linear_bwd(dyb, wb, xb, need_dx=True, dx_residual=None, need_dw=True):
    """dyb [T,N] bf16 ; wb [N,K] bf16 ; xb [T,K] bf16 -> dx fp32 [T,K] (+ residual), dw fp32 [N,K], db fp32 [N]"""
    N, K = wb.shape
    T = dyb.numel() // N
    dx = torch.empty(*dyb.shape[:-1], K, dtype=torch.float32, device=dyb.device) if need_dx else None
    dw = torch.zeros(N, K, dtype=torch.float32, device=dyb.device) if need_dw else None
    db = torch.zeros(N, dtype=torch.float32, device=dyb.device) if need_dw else None
    ws = workspace(dyb.device, "grb_linear_backward_workspace_bytes", T, N, K) if need_dw else None
    call(dyb.device, "grb_linear_backward", ptr(dyb), ptr(wb), ptr(xb), T, N, K, ptr(dx), ptr(dx_residual), ptr(dw), ptr(db), ptr(ws))
    return dx, dw, db


def _sasrec_dims(q, H, p, seed, seed_dev, layer, offsets, max_len):
    if offsets is None:
        B, L, D = q.shape
        return SasrecDims(B, L, D, H, float(p), int(seed), ptr(seed_dev), layer)
    return SasrecDims(offsets.numel() - 1, int(max_len), q.shape[-1], H, float(p), int(seed), ptr(seed_dev), layer)


def sasrec_attention_fwd(q, k, v, pad, H, p=0.0, seed=0, seed_dev=None, layer=0, offsets=None, max_len=None):
    """q, k, v [B, L, D] bf16, pad [B, L] -> (out [B, L, D] bf16, lse [B, H, L]).  With ``offsets`` ([B+1] int64 on the device) and
    ``max_len`` the batch is packed (grb_sasrec_attention_forward_jagged): q, k, v, out [T, D], pad [T], lse [H, T]."""
    dims = _sasrec_dims(q, H, p, seed, seed_dev, layer, offsets, max_len)
    out = torch.empty_like(q)
    if offsets is None:
        B, L, D = q.shape
        lse = torch.empty(B, H, L, dtype=torch.float32, device=q.device)
        call(q.device, "grb_sasrec_attention_forward", C.byref(dims), ptr(q), ptr(k), ptr(v), ptr(pad), ptr(out), ptr(lse))
    else:
        T = q.shape[0]
        lse = torch.empty(H, T, dtype=torch.float32, device=q.device)
        call(q.device, "grb_sasrec_attention_forward_jagged", C.byref(dims), ptr(offsets), T, ptr(q), ptr(k), ptr(v), ptr(pad), ptr(out),
             ptr(lse))
    return out, lse


def sasrec_attention_bwd(q, k, v, pad, out, lse, dout, H, p=0.0, seed=0, seed_dev=None, layer=0, offsets=None, max_len=None):
    """The backward of ``sasrec_attention_fwd`` -> (dq, dk, dv) shaped like q; packed with ``offsets`` and ``max_len``."""
    dims = _sasrec_dims(q, H, p, seed, seed_dev, layer, offsets, max_len)
    dq, dk, dv = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
    if offsets is None:
        call(q.device, "grb_sasrec_attention_backward", C.byref(dims), ptr(q), ptr(k), ptr(v), ptr(pad), ptr(out), ptr(lse), ptr(dout),
             ptr(dq), ptr(dk), ptr(dv))
    else:
        call(q.device, "grb_sasrec_attention_backward_jagged", C.byref(dims), ptr(offsets), q.shape[0], ptr(q), ptr(k), ptr(v), ptr(pad),
             ptr(out), ptr(lse), ptr(dout), ptr(dq), ptr(dk), ptr(dv))
    return dq, dk, dv


def linear_dact_bwd(dyb, wb, z, act, p=0.0, seed=0, seed_dev=None, site=0):
    """g[T,K] = dropmask(dyb[T,N] @ wb[N,K]) * act'(z[T,K])  (bf16)"""
    N, K = wb.shape
    T = dyb.numel() // N
    g = torch.empty_like(z)
    call(dyb.device, "grb_linear_dact_backward", ptr(dyb), ptr(wb), ptr(z), T, N, K, act, float(p), int(seed), ptr(seed_dev), site, ptr(g))
    return g


def cast_rows_bf16(x, row_scale=None, p=0.0, seed=0, seed_dev=None, site=0):
    """bf16(dropmask(x) * row_scale[:, None])"""
    D = x.shape[-1]
    T = x.numel() // D
    out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    call(x.device, "grb_cast_rows_f32_to_bf16", ptr(x), ptr(out), T, D, ptr(row_scale), float(p), int(seed), ptr(seed_dev), site)
    return out


@functools.cache
def zero_bias(n: int, device) -> torch.Tensor:
    """fp32 zeros [n] on ``device``, made once: the bias operand of a bias-free linear."""
    return torch.zeros(n, dtype=torch.float32, device=device)


def dropout_seed(p: float) -> int:
    """The host seed of a dropout call: torch's initial seed (torch.manual_seed makes a step reproducible), 0 when p is 0."""
    return torch.initial_seed() & 0x7FFFFFFFFFFFFFFF if p > 0 else 0


class StepSeeds:
    """Mixed into a module whose dropout probability is its ``_dropout_p`` (the models HSTU and SASRec, and the layers a user may
    call on their own: HSTULayer, SASRecBlock, MultiHeadAttention, PointWiseFeedForward): ``_seeds`` gives each training forward
    its (host seed, device seed), (0, None) without dropout.  The device seed is an int64 counter, made by the first training
    forward (again after ``_seed_dev = None``) and bumped by each; a CUDA graph that captures the bump draws fresh masks on every
    replay."""

    _seed_dev = None

    def _seeds(self, device):
        p = self._dropout_p
        if not (self.training and p > 0):
            return 0, None
        if self._seed_dev is None or self._seed_dev.device != device:
            self._seed_dev = torch.zeros(1, dtype=torch.int64, device=device)
            self._step_seed = dropout_seed(p)
        self._seed_dev.add_(0x9E3779B1)
        # per-forward snapshot: the backward re-derives the masks from the value THIS forward saw, even when another
        # training-mode forward has bumped the counter in between
        return self._step_seed, self._seed_dev.clone()


def matmul_f32(xb, w_t):
    """fp32 [R, N] = x W^T of bf16 operands, through the linear backward's dx GEMM, which writes fp32: xb [R, K] and w_t = W^T [K, N]
    contiguous, K and N multiples of 8 (pad W with zero rows to get there, then slice the result)."""
    y, _, _ = linear_bwd(xb, w_t, None, need_dw=False)
    return y


def ffn_fwd(xb, w1b, b1, w2b, b2, residual, row_scale, p_in, p_out, seed, seed_dev, site_hid, site_out):
    """A block's feed-forward: z = x W1^T + b1, h = drop(relu(z)) at site_hid, y = (drop(h W2^T + b2) at site_out + residual) *
    row_scale, as two fused-epilogue GEMMs on bf16 operands -> (y fp32, z, h)."""
    z, h = linear_fwd(xb, w1b, b1, 2, p_in, seed, seed_dev, site_hid)
    y = linear_residual_fwd(h, w2b, b2, residual, row_scale, p_out, seed, seed_dev, site_out)
    return y, z, h


def ffn_bwd(dy, w1b, w2b, xb, z, h, p_in, p_out, seed, seed_dev, site_hid, site_out, dx_residual=None):
    """The backward of ``ffn_fwd`` under the same dropout arguments (the cast of dy re-applies the output mask, the dact GEMM the
    hidden one): dy fp32 -> (dx fp32 (+ dx_residual), dw1, db1, dw2, db2).  The residual's gradient, dy, is the caller's."""
    dyb = cast_rows_bf16(dy, None, p_out, seed, seed_dev, site_out)
    _, dw2, db2 = linear_bwd(dyb, w2b, h, need_dx=False)
    dz = linear_dact_bwd(dyb, w2b, z, 2, p_in, seed, seed_dev, site_hid)
    dx, dw1, db1 = linear_bwd(dz, w1b, xb, dx_residual=dx_residual)
    return dx, dw1, db1, dw2, db2


# ------------------------------------------------------------------------------------------------ RQ-VAE
def rq_residual_argmin(x: torch.Tensor, codebooks: torch.Tensor, commitment: float = 0.25, want_aux: bool = True):
    """x [N, D] fp32, codebooks [levels, K, D] fp32 -> ids [N, levels] int64 (+ emb, res [N, D, levels], loss [N])."""
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
    call(x.device, "grb_rq_residual_argmin", ptr(x), ptr(cb), N, D, K, levels, float(commitment), ptr(ids), ptr(emb), ptr(res), ptr(loss),
         None)
    return ids, emb, res, loss


def rq_sinkhorn(dist: torch.Tensor, eps: float = 0.003, iters: int = 100):
    """Sinkhorn-Knopp hard assignment of the SINKHORN estimator (csrc/rq_sinkhorn.cuh): dist [B, K] fp32, 2 <= K <= 256 ->
    ids [B] int64, u [B] and v [K] fp64 (the final scalings; P = u K v)."""
    require_cuda(dist)
    require_f32(dist)
    if dist.dim() != 2:
        raise _lib.GrbError(f"genrec_b200 error -1: dist must be [B, K] (got {tuple(dist.shape)})")
    dist = dist.detach().contiguous()
    B, K = dist.shape
    ids = torch.empty(B, dtype=torch.int64, device=dist.device)
    u = torch.empty(B, dtype=torch.float64, device=dist.device)
    v = torch.empty(K, dtype=torch.float64, device=dist.device)
    ws = workspace(dist.device, "grb_rq_sinkhorn_workspace_bytes", B, K, allow_empty=B == 0)     # B = 0: nothing to do, no scratch
    call(dist.device, "grb_rq_sinkhorn", ptr(dist), B, K, float(eps), int(iters), ptr(ids), ptr(u), ptr(v), ptr(ws))
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
    call(x.device, "grb_kmeans_update", ptr(x), ptr(assign.contiguous()), B, D, k, ptr(centroids), ptr(stats[0]), ptr(stats[1]))
    return stats


def split3(x: torch.Tensor, operand: int) -> torch.Tensor:
    """fp32 [rows, K] -> bf16 [rows, 6K]: the three-term bf16 split of every value, laid out along K for the fp32-accurate GEMM
    (operand 0 = activation layout, 1 = weight layout; csrc/rowwise.cuh split3_f32_bf16_kernel)."""
    require_cuda(x)
    require_f32(x)
    x = x.detach().contiguous()
    rows, K = x.numel() // x.shape[-1], x.shape[-1]
    out = torch.empty(*x.shape[:-1], 6 * K, dtype=torch.bfloat16, device=x.device)
    call(x.device, "grb_split3_f32_to_bf16", ptr(x), ptr(out), rows, K, operand)
    return out


def linear_f32x3(x_split: torch.Tensor, w_split: torch.Tensor, act: int = 0) -> torch.Tensor:
    """y = act(x W^T) in fp32 accuracy on the tensor-core path; x_split [T, 6K], w_split [N, 6K] from split3(); act 0 none, 1 silu."""
    K6 = x_split.shape[-1]
    T, N = x_split.numel() // K6, w_split.shape[0]
    y = torch.empty(*x_split.shape[:-1], N, dtype=torch.float32, device=x_split.device)
    call(x_split.device, "grb_linear_f32x3_forward", ptr(x_split), ptr(w_split), T, N, K6 // 6, act, ptr(y))
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
    call(x_split.device, "grb_linear_f32x3_bias_forward", ptr(x_split), ptr(w_split), ptr(bias), ptr(residual), T, N, K6 // 6, act, ptr(y),
         ldy)
    return y[..., :N] if ldy != N else y


def layernorm_f32(x: torch.Tensor, g: torch.Tensor, b: torch.Tensor, eps: float) -> torch.Tensor:
    require_cuda(x)
    require_f32(x, g, b)
    x = x.detach().contiguous()
    y = torch.empty_like(x)
    call(x.device, "grb_layernorm_f32_forward", ptr(x), ptr(g.detach()), ptr(b.detach()), float(eps), x.numel() // x.shape[-1], x.shape[-1],
         ptr(y))
    return y


def hstu_layer_forward_f32(x: torch.Tensor, meta: SeqMeta, H: int, npos: int, ntime: int, split_w: dict, params) -> torch.Tensor:
    """fp32-exact forward of one HSTU block (csrc/exact_f32.cuh; hstu.py:222-280 without autocast).  ``split_w`` = the three weight
    matrices pre-split by split3(w, 1); ``params`` in PARAM_ORDER.  Forward only."""
    require_cuda(x)
    require_f32(x)
    B, L, D = x.shape
    xc = x.detach().contiguous()
    (_, proj_b, pos_t, time_t, ln1_g, ln1_b, _, ffn1_b, _, ffn2_b, ln2_g, ln2_b) = params
    join_deferred(x.device)
    seq = meta.struct()
    d = _dims(B, L, D, H, npos, ntime, 0.0, 0, None, 0)
    p = _lib.HstuLayerParamsF32(ptr(split_w["proj_w"]), ptr(proj_b.detach()), ptr(pos_t.detach()), ptr(time_t.detach()) if time_t is not None else None,
                                ptr(ln1_g.detach()), ptr(ln1_b.detach()), ptr(split_w["ffn1_w"]), ptr(ffn1_b.detach()), ptr(split_w["ffn2_w"]),
                                ptr(ffn2_b.detach()), ptr(ln2_g.detach()), ptr(ln2_b.detach()))
    ws = workspace(x.device, "grb_hstu_layer_f32_workspace_bytes", C.byref(d))
    y = torch.empty_like(xc)
    call(x.device, "grb_hstu_layer_forward_f32", C.byref(d), C.byref(p), C.byref(seq), ptr(xc), ptr(y), ptr(ws))
    return y


def adam_step(p, g, m, v, p_bf16, state, lr, beta1, beta2, eps, weight_decay, grad_scale=1.0, zero_grad=True):
    call(p.device, "grb_adam_step", ptr(p), ptr(g), ptr(m), ptr(v), ptr(p_bf16), p.numel(), ptr(state), lr, beta1, beta2, eps, weight_decay,
         grad_scale, int(zero_grad))


def rowset_mark(ids, C, flag, rows, count):
    """Add the ids in 1 .. C-1 of ``ids`` (int64, any shape, on the device) to the row set ``(flag, rows, count)`` (csrc/lazy_adam.cuh)."""
    require_cuda(ids)
    require_i64(ids)
    ids = ids.contiguous()
    call(ids.device, "grb_rowset_mark", ptr(ids), ids.numel(), C, ptr(flag), ptr(rows), ptr(count))


def rowset_mark_all(all_word):
    call(all_word.device, "grb_rowset_mark_all", ptr(all_word))


def adam_step_lazy_table(p, g, m, v, p_bf16, table_off, C, D, flag, rows, count, all_word, state, lr, beta1, beta2, eps, weight_decay,
                         grad_scale=1.0):
    """``adam_step`` with the table slot [table_off, table_off + C * D) updated on the rows of the row set only; empties the set."""
    call(p.device, "grb_adam_step_lazy_table", ptr(p), ptr(g), ptr(m), ptr(v), ptr(p_bf16), p.numel(), table_off, C, D, ptr(flag), ptr(rows),
         ptr(count), ptr(all_word), ptr(state), lr, beta1, beta2, eps, weight_decay, grad_scale)


# ------------------------------------------------------------------------------------------------ COBRA
def post_layernorm_fwd(x, g, b, eps):
    """LayerNorm of fp32 rows x [..., D] at COBRA's widths -> (y fp32, stats [T, 2])"""
    T, D = x.numel() // x.shape[-1], x.shape[-1]
    y = torch.empty_like(x)
    st = torch.empty(T, 2, dtype=torch.float32, device=x.device)
    call(x.device, "grb_post_layernorm_forward", ptr(x), ptr(g), ptr(b), float(eps), T, D, ptr(y), ptr(st))
    return y, st


def post_layernorm_bwd(dy, x, st, g):
    """-> (dx, dg, db), dg / db summed in a fixed order"""
    T, D = x.numel() // x.shape[-1], x.shape[-1]
    dx = torch.empty_like(x)
    dg, db = torch.zeros_like(g), torch.zeros_like(g)
    ws = workspace(x.device, "grb_layernorm_backward_workspace_bytes", T, D)
    call(x.device, "grb_post_layernorm_backward", ptr(dy), ptr(x), ptr(st), ptr(g), T, D, ptr(dx), ptr(dg), ptr(db), ptr(ws))
    return dx, dg, db


def cobra_pack_texts(tokens: torch.Tensor, keep: Optional[torch.Tensor] = None):
    """tokens [N, L] int64 (CUDA), keep [N] uint8 or None -> (offsets [N+1] int64, info [3] int64 on the device): text n is its
    leading non-zero tokens (none where keep is 0); info = {rows, longest text, first refused text + 1 or 0}."""
    N, L = tokens.shape
    dev = tokens.device
    lens = torch.empty(N, dtype=torch.int32, device=dev)
    offsets = torch.empty(N + 1, dtype=torch.int64, device=dev)
    info = torch.empty(3, dtype=torch.int64, device=dev)
    call(dev, "grb_cobra_pack_texts", ptr(tokens), N, L, ptr(keep), ptr(lens), ptr(offsets), ptr(info))
    return offsets, info


def cobra_text_rows(tokens: torch.Tensor, offsets: torch.Tensor, rows: int):
    """-> (token id [rows], position in its text [rows]) int64 of the packed rows"""
    N, L = tokens.shape
    tok = torch.empty(rows, dtype=torch.int64, device=tokens.device)
    pos = torch.empty(rows, dtype=torch.int64, device=tokens.device)
    call(tokens.device, "grb_cobra_text_rows", ptr(tokens), N, L, ptr(offsets), ptr(tok), ptr(pos))
    return tok, pos


def seg_layernorm_mean_fwd(offsets, x, g, b, eps):
    """x [rows, D] fp32 -> (pooled [N, D] = mean of LayerNorm(x) over each text's rows, stats [rows, 2])"""
    N, D = offsets.numel() - 1, g.numel()
    pooled = torch.empty(N, D, dtype=torch.float32, device=g.device)
    st = torch.empty(max(x.shape[0], 1), 2, dtype=torch.float32, device=g.device)
    call(g.device, "grb_seg_layernorm_mean_forward", ptr(offsets), N, ptr(x), ptr(g), ptr(b), float(eps), D, ptr(st), ptr(pooled))
    return pooled, st


def seg_layernorm_mean_bwd(offsets, x, st, g, dpooled):
    """-> (dx [rows, D], dg, db [D]), dg / db summed in a fixed order"""
    N, D = offsets.numel() - 1, g.numel()
    dx = torch.empty_like(x)
    dg, db = torch.zeros_like(g), torch.zeros_like(g)
    ws = workspace(g.device, "grb_seg_layernorm_mean_backward_workspace_bytes", N, D)
    call(g.device, "grb_seg_layernorm_mean_backward", ptr(offsets), N, ptr(x), ptr(st), ptr(g), ptr(dpooled), D, ptr(dx), ptr(dg), ptr(db),
         ptr(ws))
    return dx, dg, db


def l2norm_fwd(x, eps=1e-12):
    """F.normalize(x, dim=-1) of fp32 rows -> (y, norms [T])"""
    T, D = x.numel() // x.shape[-1], x.shape[-1]
    y = torch.empty_like(x)
    n = torch.empty(T, dtype=torch.float32, device=x.device)
    call(x.device, "grb_l2norm_forward", ptr(x), T, D, float(eps), ptr(y), ptr(n))
    return y, n


def l2norm_bwd(dy, y, norms, eps=1e-12):
    T, D = y.numel() // y.shape[-1], y.shape[-1]
    dx = torch.empty_like(y)
    call(y.device, "grb_l2norm_backward", ptr(dy), ptr(y), ptr(norms), T, D, float(eps), ptr(dx))
    return dx


def infonce_fwd_bwd(scores, lo, hi, inv_tau: float):
    """scores [Q, ld] fp32, lo / hi [Q] int64 -> (sum of the row losses [1], dscores [Q, ld] bf16 of the mean loss)"""
    Q, ld = scores.shape
    row = torch.empty(Q, dtype=torch.float32, device=scores.device)
    loss = torch.empty(1, dtype=torch.float32, device=scores.device)
    ds = torch.empty(Q, ld, dtype=torch.bfloat16, device=scores.device)
    call(scores.device, "grb_infonce_forward_backward", ptr(scores), Q, ld, ptr(lo), ptr(hi), float(inv_tau), ptr(row), ptr(loss), ptr(ds))
    return loss, ds


# ------------------------------------------------------------------------------------------------ COBRA generation
def cobra_beam_attention(q, hist_qkv, hist_len, suf_qkv, anc, S: int, H: int) -> torch.Tensor:
    """One decoder layer's self-attention of one new token per beam (grb_cobra_beam_attention).  q [B K, D] bf16 (a column view of the
    step's QKV); hist_qkv [B, Li, 3D] bf16, the prefill's QKV, whose K | V are read in place, user b's keys its first hist_len[b]
    (int32 [B]) rows; suf_qkv [steps, B K, 3D] bf16, the new tokens' QKV per step; anc [B K, S - 1] int32 (None for S = 1): the row of
    step s < S - 1 a beam descends from (step S - 1 is its own row).  -> [B K, D] bf16."""
    B, Li, D3 = hist_qkv.shape
    D = D3 // 3
    R = q.shape[0]
    K = R // B
    out = torch.empty(R, D, dtype=torch.bfloat16, device=q.device)
    ws = workspace(q.device, "grb_cobra_beam_attention_workspace_bytes", B, K, H, D // H, Li)
    call(q.device, "grb_cobra_beam_attention", ptr(q), q.stride(0), ptr(hist_qkv[..., D:]), ptr(hist_qkv[..., 2 * D:]), D3, Li, ptr(hist_len),
         ptr(suf_qkv[..., D:]), ptr(suf_qkv[..., 2 * D:]), D3, suf_qkv.stride(0), ptr(anc), S, B, K, H, D // H, ptr(out), D, ptr(ws))
    return out


def cobra_paged_attention(q, k, v, page_table, page_size: int, users, hist_len, max_keys: int, q_off, q_keys, H: int, suf_qkv=None,
                          anc=None, S: int = 0) -> torch.Tensor:
    """The attention of cobra_beam_attention for queries packed by user, history keys through a page table
    (grb_cobra_paged_attention).  q [R, D] bf16 (a column view); k / v: column views of the key rows (the pool's [pages page_size, 2D]
    for a layer, or with page_table None the prefill's QKV, page_size rows per user); users [B] int32 page-table rows (None: 0 .. B-1);
    hist_len [B] int32 keys per call row; q_off [B + 1] int32; q_keys [R] int32 history keys each query sees (<= max_keys); suf_qkv
    [steps, R, 3D] bf16, anc [R, S - 1] int32 and S suffix keys as cobra_beam_attention (S = 0: none).  -> [R, D] bf16."""
    R, D = q.shape
    B = hist_len.numel()
    ld_kv = k.stride(-2)
    pt_ld = page_table.shape[1] if page_table is not None else 1
    out = torch.empty(R, D, dtype=torch.bfloat16, device=q.device)
    ws = workspace(q.device, "grb_cobra_paged_attention_workspace_bytes", R, H, D // H, max_keys)
    sk, sv = (suf_qkv[..., D:2 * D], suf_qkv[..., 2 * D:]) if S else (None, None)
    call(q.device, "grb_cobra_paged_attention", ptr(q), q.stride(0), ptr(k), ptr(v), ld_kv, ptr(page_table), pt_ld, page_size, ptr(users),
         ptr(hist_len), max_keys, ptr(q_off), ptr(q_keys), R, ptr(sk), ptr(sv), 3 * D, suf_qkv.stride(0) if S else 0, ptr(anc), S, B, H,
         D // H, ptr(out), D, ptr(ws))
    return out


def cobra_kv_scatter(qkv, kv, page_table, page_size: int, row_user, row_pos) -> None:
    """Row r of qkv [R, 3D] bf16 writes its K | V columns into row pg(row_user[r], row_pos[r]) of kv [pages, page_size, 2D] bf16
    (grb_cobra_kv_scatter); row_user / row_pos int32 [R]."""
    R, D3 = qkv.shape
    call(qkv.device, "grb_cobra_kv_scatter", ptr(qkv), qkv.stride(0), R, D3 // 3, ptr(page_table), page_table.shape[1], page_size,
         ptr(row_user), ptr(row_pos), ptr(kv))


def cobra_beam_topk(logits, scores_in, B: int, K: int, temperature: float, anc_in=None):
    """One beam step (grb_cobra_beam_topk): logits [B K_in, V] fp32, scores_in [B, K_in] or None (zero) -> (tokens [B, K] int64,
    scores [B, K], parents [B, K] int64, anc_out [B K, S_in + 1] int32: the parent's ancestry row and the parent's own row)."""
    V = logits.shape[-1]
    K_in = logits.shape[0] // B
    S_in = 0 if anc_in is None else anc_in.shape[1]
    dev = logits.device
    tokens = torch.empty(B, K, dtype=torch.int64, device=dev)
    scores = torch.empty(B, K, dtype=torch.float32, device=dev)
    parents = torch.empty(B, K, dtype=torch.int32, device=dev)
    anc_out = torch.empty(B * K, S_in + 1, dtype=torch.int32, device=dev)
    ws = workspace(dev, "grb_cobra_beam_topk_workspace_bytes", B, K_in, V, K)
    call(dev, "grb_cobra_beam_topk", ptr(logits), ptr(scores_in), B, K_in, V, K, float(temperature), ptr(anc_in), S_in, ptr(tokens),
         ptr(scores), ptr(parents), ptr(anc_out), ptr(ws))
    return tokens, scores, parents.long(), anc_out


def cobra_dense_match(x_bf16, table_bf16):
    """x [R, D], table [N, D] bf16 -> (best [R] fp32, item [R] int64): each row's highest x . table_n, the lowest n among equal
    scores, without the [R, N] scores (grb_cobra_dense_match)."""
    R, D = x_bf16.shape
    N = table_bf16.shape[0]
    best = torch.empty(R, dtype=torch.float32, device=x_bf16.device)
    item = torch.empty(R, dtype=torch.int64, device=x_bf16.device)
    ws = workspace(x_bf16.device, "grb_cobra_dense_match_workspace_bytes", R, D, N)
    call(x_bf16.device, "grb_cobra_dense_match", ptr(x_bf16), ptr(table_bf16), R, D, N, ptr(best), ptr(item), ptr(ws))
    return best, item
