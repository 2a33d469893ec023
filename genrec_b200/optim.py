"""Flat-buffer training runtime: fused Adam + bf16 weight mirror + one NCCL all-reduce per step.

``FlatAdam(model)`` re-homes every parameter of the model as a view into ONE contiguous fp32 buffer, gives each a
``.grad`` view into one flat gradient buffer, and keeps a flat bf16 mirror that the CUDA kernels read as tensor-core
operands.  Consequences (SURVEY.md section 5, "distributed communication backend"):
  * backward kernels accumulate weight gradients straight into the flat buffer (``grad sink``) - no per-parameter
    AccumulateGrad kernels, no flatten copy before the all-reduce;
  * data-parallel training = ONE ``all_reduce(SUM)`` over the flat gradient (NCCL over NVLink/NVSwitch), the 1/world
    scale folded into the fused Adam kernel, which also refreshes the bf16 mirror and zeroes the gradient;
  * everything is CUDA-graph capturable (Adam's bias correction is ticked on the device).
Semantics = ``torch.optim.Adam(params, lr, betas, eps, weight_decay)`` followed by ``zero_grad()``.
"""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.distributed as dist

from . import functional as Fn
from ._lib import call, ptr


class FlatBuffers:
    """Device-agnostic part: one flat fp32 parameter buffer, one flat gradient buffer, one flat bf16 mirror, with every
    ``param.data`` / ``param.grad`` re-homed as a view (256-byte aligned slots).  Works on CPU tensors too, which is how the
    world_size-2 gloo tests exercise the data-parallel plumbing without a GPU."""

    def __init__(self, model: torch.nn.Module, alloc=None, pad_to: int = 64):
        """alloc(n, dtype) -> zeroed 1-D tensor (default torch.zeros on the parameters' device); pad_to: the total length is
        rounded up to a multiple of it (the peer-memory optimizer needs 8 * world)."""
        params = [p for p in model.parameters() if p.requires_grad]
        assert params, "no trainable parameters"
        dev = params[0].device
        offs, n = [], 0
        for p in params:
            offs.append(n)
            n += (p.numel() + 63) // 64 * 64          # 256-byte aligned slots (bf16 views stay 16-byte aligned)
        n = (n + pad_to - 1) // pad_to * pad_to
        self.n, self.offsets, self.params, self.device = n, offs, params, dev
        if alloc is None:
            alloc = lambda k, dt: torch.zeros(k, dtype=dt, device=dev)  # noqa: E731
        self.flat = alloc(n, torch.float32)
        self.grad = alloc(n, torch.float32)
        self.mirror = alloc(n, torch.bfloat16)
        self._mirror_view, self._grad_view = {}, {}
        with torch.no_grad():
            for p, o in zip(params, offs):
                k = p.numel()
                self.flat[o:o + k].copy_(p.detach().reshape(-1))
                p.data = self.flat[o:o + k].view(p.shape)
                p.grad = self.grad[o:o + k].view(p.shape)
                self._mirror_view[id(p)] = self.mirror[o:o + k].view(p.shape)
                self._grad_view[id(p)] = p.grad

    def mirror_of(self, p: torch.Tensor) -> torch.Tensor:
        return self._mirror_view[id(p)]

    def grad_of(self, p: torch.Tensor) -> Optional[torch.Tensor]:
        return self._grad_view.get(id(p))


def world_size(group=None) -> int:
    return dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1


def allreduce_gradients(buffers: FlatBuffers, group=None) -> float:
    """ONE all-reduce(SUM) over the flat gradient buffer; returns the scale (1/world) the optimizer must apply, i.e. DDP's
    gradient averaging (each rank back-propagates its own mean-over-valid-tokens loss, SURVEY.md section 8e)."""
    w = world_size(group)
    if w > 1:
        dist.all_reduce(buffers.grad, op=dist.ReduceOp.SUM, group=group)
    return 1.0 / w


class PeerMemory:
    """Symmetric (peer-mapped, multicast-mapped where the fabric supports it) allocations for the one-pass data-parallel optimizer
    step ``grb_dp_adam_step`` (csrc/dp_adam.cuh).  Built on ``torch.distributed._symmetric_memory`` for the rendezvous only -
    the collective itself is our kernel.  Raises if symmetric memory is unavailable; FlatAdam then keeps the NCCL all-reduce."""

    def __init__(self, device: torch.device, group=None):
        import torch.distributed._symmetric_memory as symm
        self.symm, self.device = symm, device
        self.group = group if group is not None else dist.group.WORLD
        self.world, self.rank = dist.get_world_size(self.group), dist.get_rank(self.group)
        self.handles = {}
        self.tensors = []

    def alloc(self, n: int, dtype) -> torch.Tensor:
        t = self.symm.empty(n, dtype=dtype, device=self.device)
        h = self.symm.rendezvous(t, self.group.group_name)
        t.zero_()
        self.handles[t.data_ptr()] = h
        self.tensors.append(t)
        return t

    def handle(self, t: torch.Tensor):
        return self.handles[t.data_ptr()]

    def peer_ptrs(self, t: torch.Tensor) -> torch.Tensor:
        return torch.tensor([int(x) for x in self.handle(t).buffer_ptrs], dtype=torch.int64, device=self.device)

    def multicast_ptr(self, t: torch.Tensor) -> int:
        h = self.handle(t)
        try:
            return int(h.multicast_ptr) if h.has_multicast_support(self.device.type, self.device.index) or int(h.multicast_ptr) else 0
        except Exception:  # noqa: BLE001
            return int(getattr(h, "multicast_ptr", 0) or 0)


class FlatAdam:
    def __init__(self, model: torch.nn.Module, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 0.0, process_group=None, grad_sink: bool = True, unit_loss_grad: bool = False,
                 peer_memory: Optional[bool] = None, defer_weight_grads: bool = False, lazy_table: bool = False):
        """``lazy_table=True`` updates only the rows of the HSTU item table that the step touched (lazy Adam); every other
        parameter follows the dense rule.  The touched rows of a step are the union, over every training forward since the last
        ``step()`` (grad enabled), of the input ids, the targets and the negatives that lie in 1 .. C-1: exactly the rows the
        embedding backward and the sampled head can write a gradient into.  A forward with the full head (no ``negatives``)
        touches every row 0 .. C-1.  A touched row gets this optimizer's per-element rule bit for bit (global step count and bias
        corrections included); an untouched row keeps its parameters, moments and mirror.  The marks accumulate over several
        forward / backward passes, and a training forward that is never back-propagated still marks its rows, which then step with
        a zero gradient.  Unlike ``torch.optim.SparseAdam`` / LazyAdam (``lr sqrt(bc2) / bc1 * m / (sqrt(v) + eps)``) the update
        is ``lr / bc1 * m / (sqrt(v) / sqrt(bc2) + eps)``, the dense rule; the two agree at eps = 0.  The table gradient stays a
        dense slot of the flat buffer (zero after every step); the step's work over it follows the touched rows.  Needs exactly
        one HSTU in ``model``, one process and the gradient sink; checkpoints are interchangeable with the dense optimizer's.
        ``unit_loss_grad=True`` promises that every training forward is followed by exactly one ``loss.backward()`` with
        gradient 1 (no loss scaling, no gradient accumulation through a scaled loss): the fused head then accumulates its
        parameter gradients into the flat buffer in the same pass that computes the loss.  The promise is checked on the
        device (``grb_assert_unit_scalar``).  Default False: fully general, a few microseconds slower per step.
        ``defer_weight_grads=True`` moves the dW / dE GEMMs of the backward pass to a side stream that ``step()`` joins (they are not
        on the critical path); anything else that reads ``.grad`` / the flat gradient before ``step()`` must call
        ``sync_grads()`` first.  Process-wide switch (``grb_set_defer_weight_grads``)."""
        lazy_owner = self._lazy_table_owner(model, process_group, grad_sink) if lazy_table else None
        dev0 = next(p for p in model.parameters() if p.requires_grad).device
        assert dev0.type == "cuda", "FlatAdam drives CUDA kernels; move the model to the GPU first"
        # data-parallel step: one pass over NVLink peer memory (multimem reduce + Adam + multicast parameter store, csrc/dp_adam.cuh)
        # when symmetric memory can be set up, otherwise NCCL all-reduce + the local fused Adam.  GRB_DP=nccl forces the latter.
        self.peer = None
        self.dp_mode = "single"
        w = world_size(process_group)
        want_peer = (os.environ.get("GRB_DP", "") != "nccl") if peer_memory is None else bool(peer_memory)
        if w > 1:
            self.dp_mode = "nccl-allreduce"
            if want_peer:
                try:
                    self.peer = PeerMemory(dev0, process_group)
                    self.buffers = FlatBuffers(model, alloc=self.peer.alloc, pad_to=64 * w)
                    self._peer_setup()
                    self.dp_mode = "peer-multimem" if self._mc[0] else "peer-p2p"
                except Exception as e:  # noqa: BLE001
                    if peer_memory:
                        raise
                    self.peer = None
                    self._peer_error = f"{type(e).__name__}: {e}"
        if self.peer is None:
            self.buffers = FlatBuffers(model)
        dev = self.buffers.device
        self.model, self.lr, self.betas, self.eps, self.weight_decay = model, lr, betas, eps, weight_decay
        self.group = process_group
        self.n, self.flat, self.grad, self.mirror, self.params = (self.buffers.n, self.buffers.flat, self.buffers.grad,
                                                                    self.buffers.mirror, self.buffers.params)
        self.m = torch.zeros(self.n, dtype=torch.float32, device=dev)
        self.v = torch.zeros(self.n, dtype=torch.float32, device=dev)
        self.state = torch.zeros(4, dtype=torch.float32, device=dev)
        Fn.cast_bf16(self.flat, self.mirror)
        # hand the mirror (and, optionally, the gradient sink) to the modules
        for mod in model.modules():
            if hasattr(mod, "_bf16_provider"):
                mod._bf16_provider = self.buffers.mirror_of
            if grad_sink and hasattr(mod, "_grad_sink"):
                mod._grad_sink = self.buffers.grad_of
            if grad_sink and hasattr(mod, "_unit_loss_grad"):
                mod._unit_loss_grad = bool(unit_loss_grad)
        # the kernels read the bf16 mirror, never the fp32 masters: anything that rewrites the masters behind the optimizer's
        # back (load_state_dict on resume, accelerate.load_state) must refresh it
        self._hook = model.register_load_state_dict_post_hook(lambda module, incompatible: self.refresh_mirror())
        if defer_weight_grads:
            assert grad_sink, "deferred weight gradients need the gradient sink (nothing but this optimizer consumes them)"
            Fn.set_defer_weight_grads(True)
        self.lazy_table = lazy_owner is not None
        if self.lazy_table:
            table = lazy_owner.item_embedding.weight
            self._table_rows, self._table_dim = table.shape
            self._table_off = self.buffers.offsets[next(i for i, p in enumerate(self.params) if p is table)]
            # the row set of the next step (csrc/lazy_adam.cuh): flags, the list of flagged rows, its length and the "every row" word
            self._row_flag = torch.zeros(self._table_rows, dtype=torch.int32, device=dev)
            self._row_list = torch.zeros(self._table_rows, dtype=torch.int32, device=dev)
            self._row_count = torch.zeros(2, dtype=torch.int32, device=dev)    # [0] = count, [1] = all
            lazy_owner._row_marker = self

    @staticmethod
    def _lazy_table_owner(model: torch.nn.Module, process_group, grad_sink: bool):
        """The one HSTU whose item table FlatAdam(lazy_table=True) updates lazily; ValueError for the cases it does not cover."""
        from .hstu import HSTU
        owners = [mod for mod in model.modules() if isinstance(mod, HSTU)]
        if len(owners) != 1:
            raise ValueError(f"lazy_table=True needs exactly one HSTU in the model, found {len(owners)}")
        if world_size(process_group) > 1:
            raise ValueError("lazy_table=True runs in one process; data-parallel lazy updates are not supported")
        if not grad_sink:
            raise ValueError("lazy_table=True needs grad_sink=True: the table gradient must land in the flat buffer")
        if not owners[0].item_embedding.weight.requires_grad:
            raise ValueError("lazy_table=True: the HSTU item table is frozen (requires_grad=False)")
        return owners[0]

    def _mark(self, ids: torch.Tensor) -> None:
        """Add the table rows named by ``ids`` (ids outside 1 .. C-1 are ignored) to the next step's row set."""
        Fn.rowset_mark(ids, self._table_rows, self._row_flag, self._row_list, self._row_count[0:1])

    def _mark_all(self) -> None:
        """Make the next step update every table row."""
        Fn.rowset_mark_all(self._row_count[1:2])

    def mirror_of(self, p: torch.Tensor) -> torch.Tensor:
        return self.buffers.mirror_of(p)

    def grad_of(self, p: torch.Tensor) -> Optional[torch.Tensor]:
        return self.buffers.grad_of(p)

    def world(self) -> int:
        return world_size(self.group)

    def _peer_setup(self) -> None:
        pm, b = self.peer, self.buffers
        self._sig = pm.alloc(2 * pm.world, torch.int32)
        self._epoch = torch.zeros(2, dtype=torch.int32, device=b.device)
        self._peer_ptrs = tuple(pm.peer_ptrs(t) for t in (b.grad, b.flat, b.mirror, self._sig))
        self._mc = tuple(pm.multicast_ptr(t) for t in (b.grad, b.flat, b.mirror))
        if not all(self._mc):
            self._mc = (0, 0, 0)
        torch.cuda.synchronize(b.device)
        dist.barrier(pm.group)

    def sync_grads(self) -> None:
        """Wait (on the current stream) for gradient work that was deferred to the side stream."""
        Fn.join_deferred(self.flat.device)

    def step(self) -> None:
        """world == 1: fused Adam.  world > 1: reduce + Adam + parameter broadcast in one pass over peer memory (dp_mode "peer-*"),
        or all-reduce(SUM) -> fused Adam with grad_scale = 1/world (dp_mode "nccl-allreduce"); either way the bf16 mirror is
        refreshed and the flat gradient is zero afterwards."""
        Fn.join_deferred(self.flat.device)
        if self.peer is not None:
            pg, pp, pmir, psig = self._peer_ptrs
            call(self.flat.device, "grb_dp_adam_step",
                 ptr(self.flat), ptr(self.grad), ptr(self.m), ptr(self.v), ptr(self.mirror), self._mc[0] or None, self._mc[1] or None,
                 self._mc[2] or None, ptr(pg), ptr(pp), ptr(pmir), ptr(psig), ptr(self._sig), ptr(self._epoch), self.n, self.peer.rank,
                 self.peer.world, ptr(self.state), self.lr, self.betas[0], self.betas[1], self.eps, self.weight_decay, 1.0 / self.peer.world)
            return
        if self.lazy_table:
            Fn.adam_step_lazy_table(self.flat, self.grad, self.m, self.v, self.mirror, self._table_off, self._table_rows, self._table_dim,
                                    self._row_flag, self._row_list, self._row_count[0:1], self._row_count[1:2], self.state, self.lr,
                                    self.betas[0], self.betas[1], self.eps, self.weight_decay)
            return
        scale = allreduce_gradients(self.buffers, self.group)
        Fn.adam_step(self.flat, self.grad, self.m, self.v, self.mirror, self.state, self.lr, self.betas[0], self.betas[1],
                     self.eps, self.weight_decay, scale, True)

    def zero_grad(self, set_to_none: bool = False) -> None:
        pass  # the fused step already zeroed the flat gradient

    def refresh_mirror(self) -> None:
        """Re-derive the bf16 operand mirror from the fp32 masters.  Called automatically after ``model.load_state_dict``;
        call it yourself after editing ``param.data`` in place (manual re-initialisation)."""
        Fn.cast_bf16(self.flat, self.mirror)

    def state_dict(self) -> dict:
        """Adam moments + step state (``torch.optim.Adam``-style checkpointing; parameters live in ``model.state_dict()``)."""
        m, v = self.m.clone(), self.v.clone()
        if self.peer is not None:     # each rank holds the moments of its own slice only: assemble the full vectors
            per = self.n // self.peer.world
            lo = self.peer.rank * per
            dist.all_gather_into_tensor(m, self.m[lo:lo + per].clone(), group=self.peer.group)
            dist.all_gather_into_tensor(v, self.v[lo:lo + per].clone(), group=self.peer.group)
        return {"m": m, "v": v, "state": self.state.clone(),
                "hyper": dict(lr=self.lr, betas=tuple(self.betas), eps=self.eps, weight_decay=self.weight_decay), "n": self.n}

    def load_state_dict(self, sd: dict) -> None:
        if int(sd["n"]) != self.n:
            raise ValueError(f"FlatAdam state for {sd['n']} elements does not fit this model ({self.n})")
        self.m.copy_(sd["m"]); self.v.copy_(sd["v"]); self.state.copy_(sd["state"])
        h = sd.get("hyper", {})
        self.lr, self.betas = h.get("lr", self.lr), tuple(h.get("betas", self.betas))
        self.eps, self.weight_decay = h.get("eps", self.eps), h.get("weight_decay", self.weight_decay)
        self.refresh_mirror()
