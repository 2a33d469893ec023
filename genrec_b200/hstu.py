"""Drop-in mirror of ``genrec.models.hstu`` (reference: genrec/models/hstu.py) backed by the sm_90a C-ABI library.

Same class names, constructor arguments, ``forward`` signatures, parameter names/shapes/init (SURVEY.md Appendix C),
so the reference trainers, gin files and checkpoints work unchanged.  All arithmetic of the hot path runs in our CUDA
kernels; CPU tensors raise (no fallback).

Documented deviations from the reference:
  * compute dtype is always bf16 tensor-core operands / fp32 accumulate and residual stream (what the reference does
    under ``Accelerator(mixed_precision="bf16")``); scores stay fp32 (the reference rounds Q.K^T to bf16 first);
  * in ``training`` mode with ``targets`` the [B, L, V+1] logits tensor is not materialised and ``None`` is returned in
    its place (the reference trainer discards it: hstu_trainer.py:157).  Set ``model.return_train_logits = True`` to get
    it back;
  * dropout uses a counter-based generator, so masks differ from torch's Philox stream (same distribution).
"""
from __future__ import annotations

import math
from typing import Optional, Tuple

import torch
import torch.nn as nn

from . import _lib
from . import functional as Fn
from ._lib import ensure_device, require_cuda

INT64_MAX = (1 << 63) - 1


def _temporal_bucket_ref(time_diff: torch.Tensor, num_buckets: int) -> torch.Tensor:
    """The reference bucket expression (hstu.py:376-382), used on the HOST only: to derive integer thresholds and for
    the stand-alone ``TemporalBias.forward``."""
    mag = torch.clamp(torch.abs(time_diff), min=1).float()
    return torch.clamp((torch.log(mag) / 0.693).long(), min=0, max=num_buckets - 1)


def time_bucket_thresholds() -> torch.Tensor:
    """int64[65]: thr[k] = smallest |dt| >= 1 whose un-clamped reference bucket is >= k; thr[64] = INT64_MAX.

    Derived by bisection on the reference fp32 expression itself (monotone), evaluated with torch on the CPU, so the
    kernel's integer compare ``|dt| >= thr[k]`` reproduces ``trunc(log_f32(float(|dt|)) / 0.693)`` bit-exactly,
    including the places where 0.693 != ln 2 moves a boundary (|dt| = 1023 -> bucket 10).
    """
    big = 1 << 20
    thr = [0] * 65
    for k in range(1, 64):
        lo, hi = 1, 1 << 62
        if int(_temporal_bucket_ref(torch.tensor([hi]), big)) < k:
            thr[k] = INT64_MAX
            continue
        while lo < hi:
            mid = (lo + hi) // 2
            if int(_temporal_bucket_ref(torch.tensor([mid]), big)) >= k:
                hi = mid
            else:
                lo = mid + 1
        thr[k] = lo
    thr[64] = INT64_MAX
    return torch.tensor(thr, dtype=torch.int64)


_THR_CACHE = {}


def _thresholds_on(device) -> torch.Tensor:
    key = str(device)
    if key not in _THR_CACHE:
        if "cpu" not in _THR_CACHE:
            _THR_CACHE["cpu"] = time_bucket_thresholds()
        _THR_CACHE[key] = _THR_CACHE["cpu"].to(device)
    return _THR_CACHE[key]


class RelativePositionBias(nn.Module):
    """Mirror of genrec/models/hstu.py:284-349."""

    def __init__(self, num_buckets: int = 32, max_distance: int = 128, num_heads: int = 2):
        super().__init__()
        self.num_buckets = num_buckets
        self.max_distance = max_distance
        self.num_heads = num_heads
        self.relative_attention_bias = nn.Embedding(num_buckets, num_heads)
        self._table_cache = {}
        self._uniform_cache = {}

    def _relative_position_bucket(self, relative_position: torch.Tensor) -> torch.Tensor:
        nb, md = self.num_buckets, self.max_distance
        rp = torch.clamp(relative_position, min=0)
        max_exact = nb // 2
        is_small = rp < max_exact
        large = max_exact + (torch.log(rp.float() / max_exact) / math.log(md / max_exact) * (nb - max_exact)).long()
        large = torch.clamp(large, max=nb - 1)
        return torch.where(is_small, rp, large)

    def bucket_of_delta(self, seq_len: int, device) -> torch.Tensor:
        """uint8[L]: bucket used by the reference for cell (i, j) with delta = i - j >= 0.

        The reference evaluates the bucket of ``pos[None,:] - pos[:,None]`` = j - i = -delta (hstu.py:340), clamped at 0,
        i.e. bucket 0 on the whole causal triangle (SURVEY.md section 0).  Computing it through the formula keeps this
        faithful today and makes an upstream sign fix a one-line change here (``-delta`` -> ``delta``).
        """
        key = (seq_len, str(device))
        if key not in self._table_cache:
            delta = torch.arange(seq_len)
            tbl = self._relative_position_bucket(-delta).to(torch.uint8)
            self._uniform_cache[key] = (bool((tbl == tbl[0]).all()), int(tbl[0]))
            self._table_cache[key] = tbl.to(device)
        return self._table_cache[key]

    def uniform_of(self, seq_len: int, device):
        """(all deltas share one bucket?, that bucket) for the table above - host-side, cached."""
        self.bucket_of_delta(seq_len, device)
        return self._uniform_cache[(seq_len, str(device))]

    def forward(self, seq_len: int, device: torch.device) -> torch.Tensor:
        """[H, L, L] dense bias - API parity only; the fused kernels never materialise it."""
        pos = torch.arange(seq_len, device=device)
        buckets = self._relative_position_bucket(pos.unsqueeze(0) - pos.unsqueeze(1))
        return self.relative_attention_bias(buckets).permute(2, 0, 1)


class TemporalBias(nn.Module):
    """Mirror of genrec/models/hstu.py:352-409."""

    def __init__(self, num_buckets: int = 64, num_heads: int = 2):
        super().__init__()
        self.num_buckets = num_buckets
        self.num_heads = num_heads
        self.temporal_attention_bias = nn.Embedding(num_buckets, num_heads)

    def _temporal_bucket(self, time_diff: torch.Tensor) -> torch.Tensor:
        return _temporal_bucket_ref(time_diff, self.num_buckets)

    def forward(self, timestamps: torch.Tensor) -> torch.Tensor:
        """[B, H, L, L] dense bias - API parity only (integer-threshold bucketing, identical to the kernels')."""
        thr = _thresholds_on(timestamps.device)[1:64]
        diff = (timestamps.unsqueeze(2) - timestamps.unsqueeze(1)).abs().clamp(min=1)
        buckets = torch.bucketize(diff, thr, right=True).clamp(max=self.num_buckets - 1)
        return self.temporal_attention_bias(buckets).permute(0, 3, 1, 2)


class HSTULayer(nn.Module):
    """Mirror of genrec/models/hstu.py:160-280; forward/backward = one C-ABI call each."""

    def __init__(self, embed_dim: int, num_heads: int, dropout: float, num_position_buckets: int, num_time_buckets: int,
                 max_position_distance: int, use_temporal_bias: bool):
        super().__init__()
        assert embed_dim % num_heads == 0
        self.embed_dim, self.num_heads, self.head_dim = embed_dim, num_heads, embed_dim // num_heads
        self.use_temporal_bias = use_temporal_bias
        self.projection = nn.Linear(embed_dim, 4 * embed_dim)
        self.position_bias = RelativePositionBias(num_position_buckets, max_position_distance, num_heads)
        if use_temporal_bias:
            self.temporal_bias = TemporalBias(num_time_buckets, num_heads)
        self.attn_norm = nn.LayerNorm(embed_dim)
        self.ffn = nn.Sequential(nn.Linear(embed_dim, 4 * embed_dim), nn.SiLU(), nn.Dropout(dropout),
                                 nn.Linear(4 * embed_dim, embed_dim), nn.Dropout(dropout))
        self.ffn_norm = nn.LayerNorm(embed_dim)
        self.dropout = nn.Dropout(dropout)
        self.layer_index = 0
        self._bf16 = {}            # name -> (version, tensor) : eval-mode cache of bf16 weight mirrors
        self._bf16_provider = None  # set by genrec_b200.optim.FlatAdam: param -> always-fresh bf16 view
        self._grad_sink = None      # set by FlatAdam: param -> view of the flat gradient buffer (kernels accumulate there)
        self.precision = "bf16"     # "fp32": the fp32-exact forward path (HSTU.set_precision)
        self._split = {}            # name -> (version, tensor): three-term bf16 splits of the weight matrices (fp32 path)

    def _split_weight(self, name: str, param: torch.Tensor) -> torch.Tensor:
        ent = self._split.get(name)
        if ent is None or ent[0] != param._version or ent[1].device != param.device:
            ent = (param._version, Fn.split3(param, 1))
            self._split[name] = ent
        return ent[1]

    def _run_f32(self, x: torch.Tensor, meta: Fn.SeqMeta) -> torch.Tensor:
        """fp32-exact forward (what the reference computes without autocast; 1e-5 parity target).  Forward only."""
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise RuntimeError("genrec_b200: precision='fp32' is a forward-only path (evaluation / inference / parity); "
                               "wrap the call in torch.no_grad() or train with precision='bf16'")
        if self.training and self.dropout.p > 0:
            raise RuntimeError("genrec_b200: precision='fp32' has no dropout; call model.eval()")
        sw = {"proj_w": self._split_weight("proj_w", self.projection.weight),
              "ffn1_w": self._split_weight("ffn1_w", self.ffn[0].weight),
              "ffn2_w": self._split_weight("ffn2_w", self.ffn[3].weight)}
        return Fn.hstu_layer_forward_f32(x, meta, self.num_heads, self.position_bias.num_buckets,
                                         self.temporal_bias.num_buckets if self.use_temporal_bias else 0, sw, self._params())

    # -- bf16 operand mirrors of the three weight matrices
    def _mirror(self, name: str, param: torch.Tensor) -> torch.Tensor:
        if self._bf16_provider is not None:
            return self._bf16_provider(param)
        ent = self._bf16.get(name)
        fresh = ent is not None and ent[0] == param._version and ent[1].device == param.device
        if self.training and torch.is_grad_enabled():
            fresh = False  # always re-cast while training: an optimizer step (possibly inside a CUDA graph) may have run
        if not fresh:
            ent = (param._version, Fn.cast_bf16(param, ent[1] if ent is not None and ent[1].device == param.device else None))
            self._bf16[name] = ent
        return ent[1]

    def _params(self):
        tb = self.temporal_bias.temporal_attention_bias.weight if self.use_temporal_bias else None
        return (self.projection.weight, self.projection.bias, self.position_bias.relative_attention_bias.weight, tb,
                self.attn_norm.weight, self.attn_norm.bias, self.ffn[0].weight, self.ffn[0].bias, self.ffn[3].weight,
                self.ffn[3].bias, self.ffn_norm.weight, self.ffn_norm.bias)

    def _run(self, x: torch.Tensor, meta: Fn.SeqMeta, seed: int, seed_dev) -> torch.Tensor:
        if self.precision == "fp32":
            return self._run_f32(x, meta)
        bf16w = {"proj_w": self._mirror("proj_w", self.projection.weight),
                 "ffn1_w": self._mirror("ffn1_w", self.ffn[0].weight),
                 "ffn2_w": self._mirror("ffn2_w", self.ffn[3].weight)}
        cfg = dict(H=self.num_heads, npos=self.position_bias.num_buckets,
                   ntime=self.temporal_bias.num_buckets if self.use_temporal_bias else 0,
                   p=self.dropout.p if self.training else 0.0, seed=seed, seed_dev=seed_dev, layer=self.layer_index)
        if self._grad_sink is not None and torch.is_grad_enabled():
            cfg["grad_sink"] = {n: (self._grad_sink(p) if p is not None else None) for n, p in zip(Fn.PARAM_ORDER, self._params())}
        return Fn.HstuLayerFn.apply(x, meta, cfg, bf16w, *self._params())

    def forward(self, x: torch.Tensor, causal_mask: torch.Tensor, padding_mask: torch.Tensor,
                timestamps: Optional[torch.Tensor] = None, _meta: Optional[Fn.SeqMeta] = None, _seed: int = 0,
                _seed_dev=None) -> torch.Tensor:
        """x [B,L,D] fp32, causal_mask [L,L] bool (accepted for signature parity; causality is derived from indices),
        padding_mask [B,L] bool (True = pad), timestamps [B,L] int64 or None  ->  [B,L,D] fp32."""
        require_cuda(x)
        ensure_device(x.device)
        if _meta is None:
            B, L, _ = x.shape
            ts = timestamps.contiguous() if (timestamps is not None and self.use_temporal_bias) else None
            _meta = Fn.SeqMeta(padding_mask.to(torch.uint8).contiguous(), ts,
                               self.position_bias.bucket_of_delta(L, x.device), _thresholds_on(x.device),
                               self.temporal_bias.num_buckets if self.use_temporal_bias else 0,
                               self.position_bias.num_buckets, self.position_bias.uniform_of(L, x.device))
        return self._run(x, _meta, _seed, _seed_dev)


class HSTUState:
    """Cached history of a batch of users for incremental inference (``HSTU.new_state`` / ``HSTU.extend``).

    Holds, per block, the K | V rows of every item seen so far (``kv`` [num_blocks, B, capacity, 2D] bf16), their timestamps,
    the per-user item counts and overflow flags, and each user's last final-block output (``last_hidden`` [B, D] fp32).  A state
    belongs to the parameters it was first written with: ``extend`` raises once any parameter's version counter has moved (a torch
    optimizer step, ``load_state_dict``).  ``genrec_b200.optim.FlatAdam`` writes parameters through a raw pointer and is not caught,
    so rebuild every state after any further training.  Items are never evicted: a user whose history outgrows ``capacity`` has
    the excess dropped and is flagged in ``overflowed()``; start a new state for them.
    """

    def __init__(self, batch_size: int, capacity: int, num_layers: int, embed_dim: int, device):
        if batch_size < 1:
            raise ValueError(f"batch_size must be positive, got {batch_size}")
        if not 1 <= capacity <= 16384:
            raise ValueError(f"capacity must lie in [1, 16384], got {capacity}")
        self.batch_size, self.capacity, self.num_layers = batch_size, capacity, num_layers
        self.kv = torch.zeros(num_layers, batch_size, capacity, 2 * embed_dim, dtype=torch.bfloat16, device=device)
        self.timestamps = torch.zeros(batch_size, capacity, dtype=torch.int64, device=device)
        self.lengths = torch.zeros(batch_size, dtype=torch.int32, device=device)
        self.overflow = torch.zeros(batch_size, dtype=torch.uint8, device=device)
        self.last_hidden = torch.zeros(batch_size, embed_dim, dtype=torch.float32, device=device)
        self.items_bound = 0      # host-side sum of the chunk widths extended so far: an upper bound of every user's length
        self.has_time = None      # whether the temporal bias is in use, fixed by the first extend
        self.param_versions = None

    def overflowed(self) -> torch.Tensor:
        """[B] bool on the device: users that had items dropped for lack of capacity.  Reading it on the host synchronises."""
        return self.overflow != 0

    def _struct(self) -> _lib.HstuCache:
        return _lib.HstuCache(self.batch_size, self.capacity, self.num_layers, self.kv.data_ptr(), self.timestamps.data_ptr(),
                              self.lengths.data_ptr(), self.overflow.data_ptr())


class HSTU(nn.Module):
    """Mirror of genrec/models/hstu.py:19-157."""

    def __init__(self, num_items: int, max_seq_len: int = 50, embed_dim: int = 64, num_heads: int = 2, num_blocks: int = 2,
                 dropout: float = 0.2, num_position_buckets: int = 32, num_time_buckets: int = 64,
                 max_position_distance: int = 128, use_temporal_bias: bool = True):
        super().__init__()
        self.num_items, self.max_seq_len, self.embed_dim = num_items, max_seq_len, embed_dim
        self.use_temporal_bias = use_temporal_bias
        self.item_embedding = nn.Embedding(num_items + 1, embed_dim, padding_idx=0)
        self.emb_dropout = nn.Dropout(dropout)
        self.layers = nn.ModuleList([
            HSTULayer(embed_dim, num_heads, dropout, num_position_buckets, num_time_buckets, max_position_distance,
                      use_temporal_bias) for _ in range(num_blocks)])
        for i, l in enumerate(self.layers):
            l.layer_index = i
        self.final_norm = nn.LayerNorm(embed_dim)
        self.return_train_logits = False
        self._table_bf16 = None
        self._table_split = None
        self.precision = "bf16"
        self._bf16_provider = None
        self._grad_sink = None
        self._unit_loss_grad = False   # FlatAdam(unit_loss_grad=True): head gradients go straight into the flat buffer (see HeadLossFn)
        self._step_seed = 0
        self._seed_dev = None  # device uint64 counter, bumped once per training forward (CUDA-graph-safe dropout reseeding)
        self._init_weights()

    def _init_weights(self):
        """genrec/models/hstu.py:85-97."""
        for module in self.modules():
            if isinstance(module, nn.Linear):
                nn.init.trunc_normal_(module.weight, std=0.02)
                if module.bias is not None:
                    nn.init.zeros_(module.bias)
            elif isinstance(module, nn.Embedding):
                nn.init.trunc_normal_(module.weight, std=0.02)
                if module.padding_idx is not None:
                    module.weight.data[module.padding_idx].zero_()
            elif isinstance(module, nn.LayerNorm):
                nn.init.ones_(module.weight)
                nn.init.zeros_(module.bias)

    def set_precision(self, precision: str) -> "HSTU":
        """"bf16" (default): bf16 tensor-core operands, fp32 accumulation and residual stream - the reference under
        Accelerator(mixed_precision="bf16").  "fp32": the fp32-exact forward path (split-bf16 GEMMs + fp32 attention / LayerNorm,
        csrc/exact_f32.cuh) - the reference without autocast, to 1e-5; evaluation / inference only."""
        if precision not in ("bf16", "fp32"):
            raise ValueError(f"precision must be 'bf16' or 'fp32', got {precision!r}")
        self.precision = precision
        for layer in self.layers:
            layer.precision = precision
        return self

    def _head_logits_f32(self, x: torch.Tensor) -> torch.Tensor:
        w = self.item_embedding.weight
        ent = self._table_split
        if ent is None or ent[0] != w._version or ent[1].device != w.device:
            ent = (w._version, Fn.split3(w, 1))
            self._table_split = ent
        xf = Fn.layernorm_f32(x, self.final_norm.weight, self.final_norm.bias, self.final_norm.eps)
        return Fn.linear_f32x3_bias(Fn.split3(xf, 0), ent[1], None, None, 0)

    def _table_mirror(self) -> torch.Tensor:
        w = self.item_embedding.weight
        if self._bf16_provider is not None:
            return self._bf16_provider(w)
        ent = self._table_bf16
        fresh = ent is not None and ent[0] == w._version and ent[1].device == w.device
        if self.training and torch.is_grad_enabled():
            fresh = False
        if not fresh:
            ent = (w._version, Fn.cast_bf16(w, ent[1] if ent is not None and ent[1].device == w.device else None))
            self._table_bf16 = ent
        return ent[1]

    def _seeds(self, device):
        if not (self.training and self.emb_dropout.p > 0):
            return 0, None
        if self._seed_dev is None or self._seed_dev.device != device:
            self._seed_dev = torch.zeros(1, dtype=torch.int64, device=device)
            self._step_seed = torch.initial_seed() & 0x7FFFFFFFFFFFFFFF
        self._seed_dev.add_(0x9E3779B1)  # captured by CUDA graphs: every replay draws fresh masks
        # per-forward snapshot: the backward re-derives the masks from the value THIS forward saw, even when another
        # training-mode forward has bumped the counter in between
        return self._step_seed, self._seed_dev.clone()

    def encode(self, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor]) -> torch.Tensor:
        """Embedding + all blocks (everything before final_norm).  hstu.py:117-132."""
        require_cuda(input_ids)
        ensure_device(input_ids.device)
        B, L = input_ids.shape
        seed, seed_dev = self._seeds(input_ids.device)
        p = self.emb_dropout.p if self.training else 0.0
        esink = None
        if self._grad_sink is not None and torch.is_grad_enabled():
            esink = (self._grad_sink(self.item_embedding.weight), None)
        x, pad = Fn.EmbedFn.apply(input_ids, self.item_embedding.weight, None, 1.0, 0, p, seed, seed_dev, esink)
        if len(self.layers):
            ts = timestamps.contiguous() if (timestamps is not None and self.use_temporal_bias) else None
            meta = Fn.SeqMeta(pad, ts, self.layers[0].position_bias.bucket_of_delta(L, input_ids.device),
                              _thresholds_on(input_ids.device),
                              self.layers[0].temporal_bias.num_buckets if self.use_temporal_bias else 0,
                              self.layers[0].position_bias.num_buckets,
                              self.layers[0].position_bias.uniform_of(L, input_ids.device))
            for layer in self.layers:
                layer._bf16_provider = self._bf16_provider
                x = layer(x, None, None, timestamps, _meta=meta, _seed=seed, _seed_dev=seed_dev)
        return x

    def forward(self, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor] = None,
                targets: Optional[torch.Tensor] = None) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """hstu.py:99-148.  Returns (logits [B,L,V+1] fp32 | None, loss | None)."""
        x = self.encode(input_ids, timestamps)
        if self.precision == "fp32":
            if targets is not None:
                raise RuntimeError("genrec_b200: precision='fp32' computes logits only (no loss / training)")
            return self._head_logits_f32(x), None
        table = self.item_embedding.weight
        table_bf16 = self._table_mirror()
        loss = None
        logits = None
        if targets is not None:
            hsink = None
            if self._grad_sink is not None and torch.is_grad_enabled():
                hsink = (self._grad_sink(self.final_norm.weight), self._grad_sink(self.final_norm.bias), self._grad_sink(table))
            loss = Fn.HeadLossFn.apply(x, self.final_norm.weight, self.final_norm.bias, table, table_bf16, targets,
                                       self.final_norm.eps, hsink, self._unit_loss_grad)
        if targets is None or not self.training or self.return_train_logits:
            logits = Fn.head_logits(x, self.final_norm.weight, self.final_norm.bias, table, table_bf16, self.final_norm.eps)
        return logits, loss

    @torch.no_grad()
    def last_logits(self, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[B, V+1] fp32 logits of the LAST position only (all that predict() / evaluation read): the tied-embedding GEMM runs
        on B rows instead of B*L."""
        x = self.encode(input_ids, timestamps)
        if self.precision == "fp32":
            return self._head_logits_f32(x[:, -1:, :].contiguous())[:, 0, :]
        return Fn.head_logits(x[:, -1:, :].contiguous(), self.final_norm.weight, self.final_norm.bias, self.item_embedding.weight,
                              self._table_mirror(), self.final_norm.eps)[:, 0, :]

    def new_state(self, batch_size: int, capacity: int) -> HSTUState:
        """An empty cache for ``batch_size`` users of up to ``capacity`` items each (<= 16384), on the model's device."""
        return HSTUState(batch_size, capacity, len(self.layers), self.embed_dim, self.item_embedding.weight.device)

    @torch.no_grad()
    def extend(self, state: HSTUState, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Append the non-zero ids of each row of ``input_ids`` [B, n] (with ``timestamps`` [B, n] or None), in order, to that user's
        history in ``state`` and return [B, V+1] fp32: the next-item logits of each user's latest item, as ``last_logits`` computes
        them for the left-padded concatenation of everything extended so far.  Prefilling a history is ``extend`` on a new state.

        Only the new items run through the blocks; the earlier ones are read from the cache.  Pads inside a chunk are compacted
        (positions count items): with the reference's position bias, where every causal cell uses one bucket, any padding pattern
        gives the full forward's result; with a non-uniform position-bucket table that holds for left-padded chunks only.  A user
        whose row is all padding keeps their state and gets the same logits row as from the previous call; a user with no item yet
        gets the head applied to a zero vector.  Inference only: bf16 precision, no dropout, no autograd.  CUDA-graph capturable
        after one eager call; the host-side capacity check does not run on replay, where items that do not fit are dropped and
        flagged (``state.overflowed()``)."""
        if self.precision == "fp32":
            raise RuntimeError("genrec_b200: extend runs the bf16 path only; set_precision('bf16') or use last_logits")
        if self.training and any(isinstance(m, nn.Dropout) and m.p > 0 for m in self.modules()):
            raise RuntimeError("genrec_b200: extend has no dropout; call model.eval()")
        require_cuda(input_ids)
        ensure_device(input_ids.device)
        B, n = input_ids.shape
        if B != state.batch_size or input_ids.device != state.lengths.device:
            raise ValueError(f"the state holds {state.batch_size} users on {state.lengths.device}; got input_ids {tuple(input_ids.shape)} on "
                             f"{input_ids.device}")
        if state.items_bound + n > state.capacity:
            raise ValueError(f"extending by {n} items could exceed the state's capacity ({state.items_bound} of {state.capacity} may be "
                             "used); start a new state with a larger capacity")
        use_time = timestamps is not None and self.use_temporal_bias
        versions = tuple(p._version for p in self.parameters())
        if state.param_versions is None:
            state.param_versions, state.has_time = versions, use_time
        elif state.param_versions != versions:
            raise RuntimeError("genrec_b200: the model's parameters changed after this state was written; rebuild the state")
        elif state.has_time != use_time:
            raise ValueError("timestamps must be given on every extend of a state or on none")
        dev = input_ids.device
        ids = input_ids.contiguous()
        cache = state._struct()
        positions, last_row = Fn.hstu_cache_append(cache, ids, timestamps.contiguous() if timestamps is not None else None)
        x, _ = Fn.EmbedFn.apply(ids, self.item_embedding.weight, None, 1.0, 0, 0.0, 0, None, None)
        if len(self.layers):
            rpb = self.layers[0].position_bias
            uniform, bucket0 = rpb.uniform_of(state.capacity, dev)
            pos_bucket = None if uniform else rpb.bucket_of_delta(state.capacity, dev)
            ntime = self.layers[0].temporal_bias.num_buckets if use_time else 0
            for i, layer in enumerate(self.layers):
                layer._bf16_provider = self._bf16_provider
                bf16w = {"proj_w": layer._mirror("proj_w", layer.projection.weight),
                         "ffn1_w": layer._mirror("ffn1_w", layer.ffn[0].weight),
                         "ffn2_w": layer._mirror("ffn2_w", layer.ffn[3].weight)}
                x = Fn.hstu_layer_extend(x, cache, i, positions, pos_bucket, bucket0, _thresholds_on(dev), layer.num_heads, rpb.num_buckets,
                                         ntime, bf16w, layer._params())
        latest = x[torch.arange(B, device=dev), last_row.clamp(min=0).long()]
        state.last_hidden.copy_(torch.where((last_row >= 0)[:, None], latest, state.last_hidden))
        state.items_bound += n
        return Fn.head_logits(state.last_hidden[:, None, :], self.final_norm.weight, self.final_norm.bias, self.item_embedding.weight,
                              self._table_mirror(), self.final_norm.eps)[:, 0, :]

    @torch.no_grad()
    def evaluate_batch(self, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor], targets: torch.Tensor,
                       metrics: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Leave-one-out metrics of one evaluation batch, accumulated ON THE DEVICE into ``metrics`` ([6] fp32: Recall@{1,5,10} hit
        counts, NDCG@{1,5,10} sums) - the loop of genrec/trainers/hstu_trainer.py:55-81 without per-sample ``.item()`` calls.
        Divide by the number of samples (and all-reduce across ranks) once at the end of the evaluation."""
        return Fn.eval_rank_metrics(self.last_logits(input_ids, timestamps), targets, metrics)

    @torch.no_grad()
    def predict(self, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor] = None, top_k: int = 10) -> torch.Tensor:
        """hstu.py:150-157."""
        logits, _ = self.forward(input_ids, timestamps)
        last_logits = logits[:, -1, :]
        last_logits[:, 0] = float("-inf")
        _, top_k_items = torch.topk(last_logits, top_k, dim=-1)
        return top_k_items
