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
    including the places where 0.693 != ln 2 moves a boundary (|dt| = 1023 -> bucket 10).  The search runs up to INT64_MAX:
    bucket 63 starts at |dt| ~ 9.14e18, above 2^62.
    """
    big = 1 << 20
    thr = [0] * 65
    for k in range(1, 64):
        lo, hi = 1, INT64_MAX
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


def _cached(cache: dict, key, param: torch.Tensor, make, remake: bool = False) -> torch.Tensor:
    """cache[key]: ``make(param, out)`` of the parameter's current version, remade when the version or the device changes or
    when ``remake`` is set; ``out`` is the previous result on the same device (or None), for makers that can write in place."""
    ent = cache.get(key)
    out = ent[1] if ent is not None and ent[1].device == param.device else None
    if remake or out is None or ent[0] != param._version:
        ent = (param._version, make(param, out))
        cache[key] = ent
    return ent[1]


def _split3_weight(param: torch.Tensor, _out) -> torch.Tensor:
    return Fn.split3(param, 1)


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


class HSTULayer(Fn.StepSeeds, nn.Module):
    """Mirror of genrec/models/hstu.py:160-280; forward/backward = one C-ABI call each.  HSTU passes each layer its step's seeds;
    called on its own without them, a training layer draws fresh dropout masks on each call (``StepSeeds``)."""

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

    @property
    def _dropout_p(self) -> float:
        return self.dropout.p

    def _weights(self) -> dict:
        """The three weight matrices, by their names in Fn.BF16_PARAMS."""
        return {"proj_w": self.projection.weight, "ffn1_w": self.ffn[0].weight, "ffn2_w": self.ffn[3].weight}

    def _run_f32(self, x: torch.Tensor, meta: Fn.SeqMeta) -> torch.Tensor:
        """fp32-exact forward (what the reference computes without autocast; 1e-5 parity target).  Forward only."""
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise RuntimeError("genrec_b200: precision='fp32' is a forward-only path (evaluation / inference / parity); "
                               "wrap the call in torch.no_grad() or train with precision='bf16'")
        if self.training and self.dropout.p > 0:
            raise RuntimeError("genrec_b200: precision='fp32' has no dropout; call model.eval()")
        sw = {n: _cached(self._split, n, w, _split3_weight) for n, w in self._weights().items()}
        return Fn.hstu_layer_forward_f32(x, meta, self.num_heads, self.position_bias.num_buckets,
                                         self.temporal_bias.num_buckets if self.use_temporal_bias else 0, sw, self._params())

    def _mirror(self, name: str, param: torch.Tensor) -> torch.Tensor:
        if self._bf16_provider is not None:
            return self._bf16_provider(param)
        # always re-cast while training: an optimizer step (possibly inside a CUDA graph) may have run
        return _cached(self._bf16, name, param, Fn.cast_bf16, remake=self.training and torch.is_grad_enabled())

    def _bf16_weights(self) -> dict:
        """bf16 operand mirrors of the three weight matrices."""
        return {n: self._mirror(n, w) for n, w in self._weights().items()}

    def _seq_meta(self, pad_u8: torch.Tensor, timestamps: Optional[torch.Tensor], L: int, device) -> Fn.SeqMeta:
        """Sequence metadata of a batch for this block's bias configuration (every block of an HSTU shares it)."""
        ts = timestamps.contiguous() if (timestamps is not None and self.use_temporal_bias) else None
        return Fn.SeqMeta(pad_u8, ts, self.position_bias.bucket_of_delta(L, device), _thresholds_on(device),
                          self.temporal_bias.num_buckets if self.use_temporal_bias else 0, self.position_bias.num_buckets,
                          self.position_bias.uniform_of(L, device))

    def _seq_meta_jagged(self, pad_u8: torch.Tensor, timestamps: Optional[torch.Tensor], offsets: torch.Tensor, max_len: int,
                         device) -> Fn.SeqMeta:
        """``_seq_meta`` of a packed batch: pad_u8 / timestamps [T], offsets [B+1] on the device, the index matrix [T, ld]."""
        ts = timestamps.contiguous() if (timestamps is not None and self.use_temporal_bias) else None
        return Fn.SeqMeta(pad_u8, ts, self.position_bias.bucket_of_delta(max_len, device), _thresholds_on(device),
                          self.temporal_bias.num_buckets if self.use_temporal_bias else 0, self.position_bias.num_buckets,
                          self.position_bias.uniform_of(max_len, device), offsets=offsets, max_len=max_len)

    def _params(self):
        tb = self.temporal_bias.temporal_attention_bias.weight if self.use_temporal_bias else None
        return (self.projection.weight, self.projection.bias, self.position_bias.relative_attention_bias.weight, tb,
                self.attn_norm.weight, self.attn_norm.bias, self.ffn[0].weight, self.ffn[0].bias, self.ffn[3].weight,
                self.ffn[3].bias, self.ffn_norm.weight, self.ffn_norm.bias)

    def _run(self, x: torch.Tensor, meta: Fn.SeqMeta, seed: int, seed_dev) -> torch.Tensor:
        if self.precision == "fp32":
            return self._run_f32(x, meta)
        bf16w = self._bf16_weights()
        cfg = dict(H=self.num_heads, npos=self.position_bias.num_buckets,
                   ntime=self.temporal_bias.num_buckets if self.use_temporal_bias else 0,
                   p=self.dropout.p if self.training else 0.0, seed=seed, seed_dev=seed_dev, layer=self.layer_index)
        if self._grad_sink is not None and torch.is_grad_enabled():
            cfg["grad_sink"] = {n: (self._grad_sink(p) if p is not None else None) for n, p in zip(Fn.PARAM_ORDER, self._params())}
        return Fn.HstuLayerFn.apply(x, meta, cfg, bf16w, *self._params())

    def forward(self, x: torch.Tensor, causal_mask: torch.Tensor, padding_mask: torch.Tensor,
                timestamps: Optional[torch.Tensor] = None, _meta: Optional[Fn.SeqMeta] = None, _seed: Optional[int] = None,
                _seed_dev=None) -> torch.Tensor:
        """x [B,L,D] fp32, causal_mask [L,L] bool (accepted for signature parity; causality is derived from indices),
        padding_mask [B,L] bool (True = pad), timestamps [B,L] int64 or None  ->  [B,L,D] fp32.  _seed / _seed_dev: the step's
        seeds (HSTU passes them); None: the layer's own."""
        require_cuda(x)
        ensure_device(x.device)
        if _seed is None:
            _seed, _seed_dev = self._seeds(x.device)
        if _meta is None:
            _meta = self._seq_meta(padding_mask.to(torch.uint8).contiguous(), timestamps, x.shape[1], x.device)
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


class HSTUPool:
    """Paged history cache of many users for serving (``HSTU.new_pool`` / ``HSTU.extend_users`` / ``HSTUPool.release``).

    Every block's K | V rows live in ``num_pages`` pages of ``page_size`` items shared by all users (``kv`` [num_blocks, num_pages,
    page_size, 2D] bf16, ``timestamps`` [num_pages, page_size]); ``page_table`` [max_users, ceil(max_items / page_size)] maps a
    user's item p to page ``page_table[u, p // page_size]``.  Pages are handed out on the device as a user's items arrive and come
    back on ``release``, so memory follows the items actually cached.  A user holds at most ``max_items`` items; items beyond that,
    or that find no free page, are dropped and flag the user in ``overflowed()``.  ``errors()`` has bit ``ERR_USER_RANGE`` set after
    a call named a user outside [0, max_users) and ``ERR_USER_REPEAT`` after a call named a user twice (those rows count as padding).
    Like ``HSTUState``, a pool belongs to the parameters it was first written with.

    The host keeps a conservative bound of each user's items (the sum of the chunk widths since the user's last release) and of the
    pages in use, and refuses an eager call with ``users`` on the CPU that could break a limit.  Calls with ``users`` on the device
    (CUDA graphs) skip those checks and do not update the bounds; the device rules above decide instead.
    """
    ERR_USER_RANGE, ERR_USER_REPEAT = 1, 2

    def __init__(self, max_users: int, num_pages: int, page_size: int, max_items: int, num_layers: int, embed_dim: int, device):
        if max_users < 1 or num_pages < 1:
            raise ValueError(f"max_users and num_pages must be positive, got {max_users}, {num_pages}")
        if page_size < 64 or page_size % 64:
            raise ValueError(f"page_size must be a positive multiple of 64 (the attention's key tile), got {page_size}")
        if not 1 <= max_items <= 16384:
            raise ValueError(f"max_items must lie in [1, 16384], got {max_items}")
        self.max_users, self.num_pages, self.page_size, self.max_items = max_users, num_pages, page_size, max_items
        self.num_layers = num_layers
        self.kv = torch.zeros(num_layers, num_pages, page_size, 2 * embed_dim, dtype=torch.bfloat16, device=device)
        self.timestamps = torch.zeros(num_pages, page_size, dtype=torch.int64, device=device)
        self.page_table = torch.zeros(max_users, -(-max_items // page_size), dtype=torch.int32, device=device)
        self.lengths = torch.zeros(max_users, dtype=torch.int32, device=device)
        self.overflow = torch.zeros(max_users, dtype=torch.uint8, device=device)
        self.free_stack = torch.arange(num_pages - 1, -1, -1, dtype=torch.int32, device=device)   # page 0 goes out first
        self.free_top = torch.full((1,), num_pages, dtype=torch.int32, device=device)
        self.error_bits = torch.zeros(1, dtype=torch.int32, device=device)
        self.row_of = torch.full((max_users,), (1 << 31) - 1, dtype=torch.int32, device=device)
        # each user's last final-block output; the extra last row stays zero and stands in for rejected rows
        self.last_hidden = torch.zeros(max_users + 1, embed_dim, dtype=torch.float32, device=device)
        self.items_bound = torch.zeros(max_users, dtype=torch.int64)   # host
        self.pages_bound = 0
        self.has_time = None
        self.param_versions = None

    def overflowed(self) -> torch.Tensor:
        """[max_users] bool on the device: users that had items dropped.  Reading it on the host synchronises."""
        return self.overflow != 0

    def pages_free(self) -> torch.Tensor:
        """0-dim int32 on the device: pages not held by any user."""
        return self.free_top[0]

    def errors(self) -> torch.Tensor:
        """0-dim int32 on the device: ERR_USER_RANGE | ERR_USER_REPEAT bits of every call so far."""
        return self.error_bits[0]

    def _pages(self, items: torch.Tensor) -> torch.Tensor:
        return (items + self.page_size - 1) // self.page_size

    def _host_users(self, users: torch.Tensor) -> torch.Tensor:
        if users.dim() != 1 or users.numel() == 0:
            raise ValueError(f"users must be a non-empty 1-D tensor, got shape {tuple(users.shape)}")
        u = users.long()
        if bool(((u < 0) | (u >= self.max_users)).any()):
            raise ValueError(f"users out of range [0, {self.max_users}): {u[(u < 0) | (u >= self.max_users)].tolist()[:8]}")
        if torch.unique(u).numel() != u.numel():
            raise ValueError("users must be distinct within a call")
        return u

    def _check_room(self, u: torch.Tensor, n: int):
        """Host refusal of a chunk of width n for CPU users u; returns the bound update to apply once the call is launched."""
        old = self.items_bound[u]
        new = old + n
        if bool((new > self.max_items).any()):
            bad = u[new > self.max_items].tolist()[:8]
            raise ValueError(f"extending by {n} items could exceed max_items ({self.max_items}) for users {bad}; release them first")
        pages = self.pages_bound + int(self._pages(new).sum() - self._pages(old).sum())
        if pages > self.num_pages:
            raise ValueError(f"extending by {n} items could need {pages} pages of the pool's {self.num_pages}; release users first")
        return new, pages

    def release(self, users) -> None:
        """Forget ``users`` (distinct, any subset): their pages return to the pool, their lengths, overflow flags and last outputs
        become zero, and the next ``extend_users`` starts their histories afresh."""
        users = torch.as_tensor(users, dtype=torch.int64) if not isinstance(users, torch.Tensor) else users
        dev = self.lengths.device
        if not users.is_cuda:
            u = self._host_users(users)
            self.pages_bound -= int(self._pages(self.items_bound[u]).sum())
            self.items_bound[u] = 0
            users = u.to(dev)
        Fn.hstu_pool_release(self._struct(), users.long(), self.last_hidden)

    def _struct(self) -> _lib.HstuPool:
        return _lib.HstuPool(self.max_users, self.num_layers, self.page_size, self.num_pages, self.max_items, self.kv.data_ptr(),
                             self.timestamps.data_ptr(), self.page_table.data_ptr(), self.lengths.data_ptr(), self.overflow.data_ptr(),
                             self.free_stack.data_ptr(), self.free_top.data_ptr(), self.error_bits.data_ptr(), self.row_of.data_ptr())


class HSTU(Fn.StepSeeds, nn.Module):
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
        self._table_casts = {}     # "bf16" / "split" -> (version, tensor): the embedding table's operand copies
        self.precision = "bf16"
        self._bf16_provider = None
        self._grad_sink = None
        self._unit_loss_grad = False   # FlatAdam(unit_loss_grad=True): head gradients go straight into the flat buffer (see HeadLossFn)
        self._row_marker = None        # set by FlatAdam(lazy_table=True): training forwards mark the item-table rows they touch
        self._init_weights()

    @property
    def _dropout_p(self) -> float:
        return self.emb_dropout.p

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
        split = _cached(self._table_casts, "split", self.item_embedding.weight, _split3_weight)
        xf = Fn.layernorm_f32(x, self.final_norm.weight, self.final_norm.bias, self.final_norm.eps)
        return Fn.linear_f32x3_bias(Fn.split3(xf, 0), split, None, None, 0)

    def _table_mirror(self) -> torch.Tensor:
        w = self.item_embedding.weight
        if self._bf16_provider is not None:
            return self._bf16_provider(w)
        return _cached(self._table_casts, "bf16", w, Fn.cast_bf16, remake=self.training and torch.is_grad_enabled())

    def _marks_rows(self) -> bool:
        """A training forward under FlatAdam(lazy_table=True): the gradient sink is set and grad is enabled (as for esink / hsink)."""
        return self._row_marker is not None and self._grad_sink is not None and torch.is_grad_enabled()

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
        if self._marks_rows():
            self._row_marker._mark(input_ids)
        if len(self.layers):
            meta = self.layers[0]._seq_meta(pad, timestamps, L, input_ids.device)
            for layer in self.layers:
                layer._bf16_provider = self._bf16_provider
                x = layer(x, None, None, timestamps, _meta=meta, _seed=seed, _seed_dev=seed_dev)
        return x

    def forward(self, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor] = None, targets: Optional[torch.Tensor] = None, *,
                negatives: Optional[torch.Tensor] = None, log_q: Optional[torch.Tensor] = None
                ) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """hstu.py:99-148.  Returns (logits [B,L,V+1] fp32 | None, loss | None).

        ``negatives`` ([N] int64 on the model's device, shared by every token; ``data.sample_negatives``) switches the loss to the
        sampled softmax with the logQ correction ``log_q`` ([V+1] fp32 or None): its cost does not depend on the catalog size.  It
        needs ``targets`` and returns ``(None, loss)``; evaluation and serving always score the full catalog."""
        if negatives is None and log_q is not None:
            raise ValueError("log_q corrects the sampled softmax: pass negatives with it")
        if negatives is not None and targets is None:
            raise ValueError("negatives select the sampled-softmax loss, which needs targets")
        x = self.encode(input_ids, timestamps)
        if self.precision == "fp32":
            if targets is not None:
                raise RuntimeError("genrec_b200: precision='fp32' computes logits only (no loss / training)")
            return self._head_logits_f32(x), None
        return self._head(x, targets, negatives, log_q)

    def _head(self, x: torch.Tensor, targets: Optional[torch.Tensor], negatives: Optional[torch.Tensor], log_q: Optional[torch.Tensor]
              ) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """The bf16 head of ``forward`` on x [B, L, D]: (logits [B, L, V+1] | None, loss | None) under forward's rules."""
        table = self.item_embedding.weight
        table_bf16 = self._table_mirror()
        loss = None
        logits = None
        if targets is not None:
            hsink = None
            if self._grad_sink is not None and torch.is_grad_enabled():
                hsink = (self._grad_sink(self.final_norm.weight), self._grad_sink(self.final_norm.bias), self._grad_sink(table))
            if negatives is not None:
                loss = Fn.SampledHeadLossFn.apply(x, self.final_norm.weight, self.final_norm.bias, table, table_bf16, targets, negatives,
                                                  log_q, self.final_norm.eps, hsink, self._unit_loss_grad)
                if self._marks_rows():
                    self._row_marker._mark(targets)
                    self._row_marker._mark(negatives)
                return None, loss
            loss = Fn.HeadLossFn.apply(x, self.final_norm.weight, self.final_norm.bias, table, table_bf16, targets,
                                       self.final_norm.eps, hsink, self._unit_loss_grad)
            if self._marks_rows():
                self._row_marker._mark_all()       # the full softmax writes a gradient into every row, 0 included
        if targets is None or not self.training or self.return_train_logits:
            logits = Fn.head_logits(x, self.final_norm.weight, self.final_norm.bias, table, table_bf16, self.final_norm.eps)
        return logits, loss

    def _check_jagged(self, what: str, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int,
                      timestamps: Optional[torch.Tensor]) -> torch.Tensor:
        """Argument check of a packed batch (before any launch) -> offsets on the model's device.  More than 65535 sequences are
        refused with ValueError wherever the offsets live.  CPU offsets are refused with
        ValueError unless offsets[0] == 0, they never decrease, no length exceeds max_len and offsets[B] <= T; device offsets are
        not read on the host (CUDA graphs), and the kernels keep a malformed one inside the T rows."""
        if self.precision == "fp32":
            raise RuntimeError(f"genrec_b200: {what} runs the bf16 path only; set_precision('bf16')")
        if timestamps is not None and tuple(timestamps.shape) != (input_ids.numel(),):
            raise ValueError(f"{what}: timestamps must be [{input_ids.numel()}] like input_ids, got {tuple(timestamps.shape)}")
        return Fn.check_jagged_batch(what, input_ids, offsets, max_len, 16384)

    def encode_jagged(self, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int, timestamps: Optional[torch.Tensor] = None
                      ) -> torch.Tensor:
        """``encode`` of a packed batch: input_ids / timestamps [T], offsets [B+1] int64 on the device (sequence b = rows
        offsets[b] .. offsets[b+1]-1), max_len >= every length -> [T, D] fp32.  No pads are computed: the blocks run on T rows."""
        T = input_ids.numel()
        seed, seed_dev = self._seeds(input_ids.device)
        p = self.emb_dropout.p if self.training else 0.0
        esink = None
        if self._grad_sink is not None and torch.is_grad_enabled():
            esink = (self._grad_sink(self.item_embedding.weight), None)
        # HSTU has no position table, so the embedding of a packed batch is that of one [1, T] row
        x, pad = Fn.EmbedFn.apply(input_ids.view(1, T), self.item_embedding.weight, None, 1.0, 0, p, seed, seed_dev, esink)
        if self._marks_rows():
            self._row_marker._mark(input_ids)
        x = x.view(T, self.embed_dim)
        if len(self.layers):
            meta = self.layers[0]._seq_meta_jagged(pad.view(T), timestamps, offsets, max_len, input_ids.device)
            for layer in self.layers:
                layer._bf16_provider = self._bf16_provider
                x = layer(x, None, None, timestamps, _meta=meta, _seed=seed, _seed_dev=seed_dev)
        return x

    def forward_jagged(self, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int, timestamps: Optional[torch.Tensor] = None,
                       targets: Optional[torch.Tensor] = None, *, negatives: Optional[torch.Tensor] = None,
                       log_q: Optional[torch.Tensor] = None) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
        """``forward`` on a packed batch (``data.pack_jagged``): input_ids / timestamps / targets [T] int64, offsets [B+1] int64
        (sequence b = rows offsets[b] .. offsets[b+1]-1; rows from offsets[B] to T are idle, id 0 and target 0), max_len >= every
        length (<= 16384).  Returns (logits [T, V+1] fp32 | None, loss | None) under ``forward``'s rules (dropout, sampled head,
        FlatAdam's gradient sinks, unit_loss_grad, lazy_table row marks).  Every stage runs on the T rows, none on padding.

        HSTU has no absolute position embedding, so each token computes what it computes in the left-padded batch of the same users;
        only dropout differs: its masks are keyed by token row, so a packed batch draws other masks than the padded one.  With
        offsets on the CPU the batch is checked before any launch (ValueError); offsets on the device are not read on the host, so a
        step with fixed (B, T, max_len) can be captured in a CUDA graph and replayed with new offsets, ids and targets.  bf16 only."""
        if negatives is None and log_q is not None:
            raise ValueError("log_q corrects the sampled softmax: pass negatives with it")
        if negatives is not None and targets is None:
            raise ValueError("negatives select the sampled-softmax loss, which needs targets")
        T = input_ids.numel()
        if targets is not None and tuple(targets.shape) != (T,):
            raise ValueError(f"forward_jagged: targets must be [{T}] like input_ids, got {tuple(targets.shape)}")
        offsets = self._check_jagged("forward_jagged", input_ids, offsets, max_len, timestamps)
        x = self.encode_jagged(input_ids, offsets, max_len, timestamps)
        logits, loss = self._head(x.view(1, T, self.embed_dim), targets, negatives, log_q)
        return (logits.view(T, -1) if logits is not None else None), loss

    @torch.no_grad()
    def evaluate_batch_jagged(self, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int, timestamps: Optional[torch.Tensor],
                              targets: torch.Tensor, metrics: Optional[torch.Tensor] = None, *, exclude: Optional[torch.Tensor] = None,
                              want_ranks: bool = False):
        """``evaluate_batch`` on a packed batch (input_ids / timestamps [T], offsets [B+1], max_len as in ``forward_jagged``; targets
        [B] the held-out item of each sequence): each sequence is ranked from its last row, offsets[b+1] - 1, and the metrics are
        accumulated into ``metrics`` on the device.  A sequence of length 0 is not ranked (rank 0, adds nothing).  With
        ``want_ranks`` it returns (metrics, ranks [B] int32)."""
        B, T = offsets.numel() - 1, input_ids.numel()
        if tuple(targets.shape) != (B,):
            raise ValueError(f"evaluate_batch_jagged: targets must be [{B}] (one per sequence), got {tuple(targets.shape)}")
        offsets = self._check_jagged("evaluate_batch_jagged", input_ids, offsets, max_len, timestamps)
        Fn.check_exclude_arg(exclude, B, input_ids.device)
        x = self.encode_jagged(input_ids, offsets, max_len, timestamps)
        last = (offsets[1:] - 1).clamp(0, T - 1)
        ranked = torch.where(offsets[1:] > offsets[:-1], targets, torch.zeros_like(targets))
        return Fn.head_rank_metrics(x.index_select(0, last), self.final_norm.weight, self.final_norm.bias, self._table_mirror(),
                                    self.final_norm.eps, ranked, metrics, exclude, want_ranks)

    @torch.no_grad()
    def last_logits(self, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor] = None) -> torch.Tensor:
        """[B, V+1] fp32 logits of the LAST position only (all that predict() / evaluation read): the tied-embedding GEMM runs
        on B rows instead of B*L."""
        x = self.encode(input_ids, timestamps)
        if self.precision == "fp32":
            return self._head_logits_f32(x[:, -1:, :].contiguous())[:, 0, :]
        return Fn.head_logits(x[:, -1:, :].contiguous(), self.final_norm.weight, self.final_norm.bias, self.item_embedding.weight,
                              self._table_mirror(), self.final_norm.eps)[:, 0, :]

    @torch.no_grad()
    def recommend(self, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor] = None, top_k: int = 10,
                  exclude: Optional[torch.Tensor] = None) -> Fn.TopItems:
        """The ``top_k`` (1..64) best next items of each row, best first, as ``TopItems(scores [B, top_k] fp32, items [B, top_k]
        int64)``, without forming the [B, V+1] logits: the head runs on the last position only and keeps each row's best items as it
        scores the table.  The scores are bit-identical to ``last_logits``; item 0 and the ids of the row's ``exclude`` ([B, E]
        int64 on the model's device, any order, E <= 16384) never appear; equal scores go to the lower item id; slots without an
        eligible item hold (-inf, 0).  bf16 precision only."""
        self._check_topk("recommend", top_k, exclude, input_ids.shape[0], input_ids.device)
        x = self.encode(input_ids, timestamps)
        return self._hidden_topk(x[:, -1, :], top_k, exclude)

    @torch.no_grad()
    def retrieve(self, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor] = None, num_candidates: int = 500,
                 exclude: Optional[torch.Tensor] = None) -> Fn.TopItems:
        """The retrieval stage of serving: ``recommend`` for up to 2048 items per row.  The ``num_candidates`` (1..2048) best next
        items of each row, best first, as ``TopItems(scores [B, num_candidates] fp32, items [B, num_candidates] int64)``, without
        forming the [B, V+1] logits, under ``recommend``'s rules (scores bit-identical to ``last_logits``, item 0 and ``exclude``
        ids left out, ties to the lower id, (-inf, 0) where no eligible item is left).  bf16 precision only."""
        self._check_candidates("retrieve", num_candidates, exclude, input_ids.shape[0], input_ids.device)
        x = self.encode(input_ids, timestamps)
        return self._hidden_select(x[:, -1, :], None, num_candidates, exclude)

    @torch.no_grad()
    def recommend_jagged(self, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int, timestamps: Optional[torch.Tensor] = None,
                         top_k: int = 10, exclude: Optional[torch.Tensor] = None) -> Fn.TopItems:
        """``recommend`` on a packed batch (input_ids / timestamps [T], offsets [B+1], max_len as in ``forward_jagged``): one row of
        ``TopItems`` per sequence, selected from the head of its last row, offsets[b+1] - 1.  A sequence of length 0 gets the head
        of a zero vector, as ``extend`` gives a user with no items.  The uncached counterpart of a packed prefill."""
        offsets = self._check_jagged("recommend_jagged", input_ids, offsets, max_len, timestamps)
        self._check_topk("recommend_jagged", top_k, exclude, offsets.numel() - 1, input_ids.device)
        x = self.encode_jagged(input_ids, offsets, max_len, timestamps)
        return self._hidden_topk(Fn.last_rows_jagged(x, offsets), top_k, exclude)

    @torch.no_grad()
    def retrieve_jagged(self, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int, timestamps: Optional[torch.Tensor] = None,
                        num_candidates: int = 500, exclude: Optional[torch.Tensor] = None) -> Fn.TopItems:
        """``retrieve`` on a packed batch, under ``recommend_jagged``'s rules: up to 2048 items per sequence."""
        offsets = self._check_jagged("retrieve_jagged", input_ids, offsets, max_len, timestamps)
        self._check_candidates("retrieve_jagged", num_candidates, exclude, offsets.numel() - 1, input_ids.device)
        x = self.encode_jagged(input_ids, offsets, max_len, timestamps)
        return self._hidden_select(Fn.last_rows_jagged(x, offsets), None, num_candidates, exclude)

    def _check_topk(self, what: str, top_k: int, exclude: Optional[torch.Tensor], rows: int, device) -> None:
        if self.precision == "fp32":
            raise RuntimeError(f"genrec_b200: {what} runs the bf16 path only; set_precision('bf16') or use last_logits")
        Fn.check_topk_args(top_k, exclude, rows, device)

    def _check_candidates(self, what: str, num_candidates: int, exclude: Optional[torch.Tensor], rows: int, device) -> None:
        if self.precision == "fp32":
            raise RuntimeError(f"genrec_b200: {what} runs the bf16 path only; set_precision('bf16') or use last_logits")
        Fn.check_candidates_args(num_candidates, exclude, rows, device)

    def _check_serving_topk(self, what: str, top_k: Optional[int], num_candidates: Optional[int], exclude: Optional[torch.Tensor],
                            rows: int, device) -> None:
        """Argument check of the top_k / num_candidates / exclude keywords of extend and extend_users (before any launch)."""
        if top_k is not None and num_candidates is not None:
            raise ValueError(f"{what}: give top_k or num_candidates, not both")
        if num_candidates is not None:
            self._check_candidates(what, num_candidates, exclude, rows, device)
            return
        if top_k is None:
            if exclude is not None:
                raise ValueError(f"{what}: exclude needs top_k or num_candidates")
            return
        self._check_topk(what, top_k, exclude, rows, device)

    def _hidden_topk(self, hidden: torch.Tensor, top_k: int, exclude: Optional[torch.Tensor]) -> Fn.TopItems:
        return Fn.head_topk(hidden, self.final_norm.weight, self.final_norm.bias, self._table_mirror(), self.final_norm.eps, top_k,
                            exclude)

    def _hidden_select(self, hidden: torch.Tensor, top_k: Optional[int], num_candidates: Optional[int],
                       exclude: Optional[torch.Tensor]):
        """TopItems of ``hidden`` for top_k or num_candidates, or the logits when neither is given."""
        if top_k is not None:
            return self._hidden_topk(hidden, top_k, exclude)
        if num_candidates is not None:
            return Fn.head_candidates(hidden, self.final_norm.weight, self.final_norm.bias, self._table_mirror(), self.final_norm.eps,
                                      num_candidates, exclude)
        return self._hidden_logits(hidden)

    def new_state(self, batch_size: int, capacity: int) -> HSTUState:
        """An empty cache for ``batch_size`` users of up to ``capacity`` items each (<= 16384), on the model's device."""
        return HSTUState(batch_size, capacity, len(self.layers), self.embed_dim, self.item_embedding.weight.device)

    @torch.no_grad()
    def extend(self, state: HSTUState, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor] = None, *, top_k: Optional[int] = None,
               num_candidates: Optional[int] = None, exclude: Optional[torch.Tensor] = None):
        """Append the non-zero ids of each row of ``input_ids`` [B, n] (with ``timestamps`` [B, n] or None), in order, to that user's
        history in ``state`` and return [B, V+1] fp32: the next-item logits of each user's latest item, as ``last_logits`` computes
        them for the left-padded concatenation of everything extended so far.  Prefilling a history is ``extend`` on a new state.
        With ``top_k`` (1..64) it returns ``TopItems`` of the same rows instead, as ``recommend`` selects them from those logits
        (``exclude`` [B, E] int64: ids left out per row), and the logits are never formed; ``num_candidates`` (1..2048, not together
        with ``top_k``) does the same for up to 2048 items, as ``retrieve`` selects them.

        Only the new items run through the blocks; the earlier ones are read from the cache.  Pads inside a chunk are compacted
        (positions count items): with the reference's position bias, where every causal cell uses one bucket, any padding pattern
        gives the full forward's result; with a non-uniform position-bucket table that holds for left-padded chunks only.  A user
        whose row is all padding keeps their state and gets the same logits row as from the previous call; a user with no item yet
        gets the head applied to a zero vector.  Inference only: bf16 precision, no dropout, no autograd.  CUDA-graph capturable
        after one eager call; the host-side capacity check does not run on replay, where items that do not fit are dropped and
        flagged (``state.overflowed()``)."""
        self._check_extend_mode("extend")
        require_cuda(input_ids)
        ensure_device(input_ids.device)
        B, n = input_ids.shape
        if B != state.batch_size or input_ids.device != state.lengths.device:
            raise ValueError(f"the state holds {state.batch_size} users on {state.lengths.device}; got input_ids {tuple(input_ids.shape)} on "
                             f"{input_ids.device}")
        self._check_serving_topk("extend", top_k, num_candidates, exclude, B, input_ids.device)
        return self._extend_state(state, input_ids, timestamps, None, n, n, top_k, num_candidates, exclude)

    @torch.no_grad()
    def extend_jagged(self, state: HSTUState, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int,
                      timestamps: Optional[torch.Tensor] = None, *, top_k: Optional[int] = None, num_candidates: Optional[int] = None,
                      exclude: Optional[torch.Tensor] = None):
        """``extend`` on a packed chunk: input_ids / timestamps [T] int64, offsets [B+1] int64 with B = ``state.batch_size``
        (sequence b = rows offsets[b] .. offsets[b+1]-1 appends to user b; rows from offsets[B] to T are idle), max_len >= every
        length and <= the state's capacity.  Returns what ``extend`` returns for the padded [B, max_len] chunk holding the same
        items per user, bit for bit, and leaves the state as that call does; only the T rows run through the blocks, none of them
        padding.  An empty sequence leaves its user untouched.  Ids equal to 0 inside a sequence still count as pads.  A packed chunk
        has no pads ahead of a user's items, so prefilling packed histories gives ``last_logits`` of the left-padded batch for
        every position-bucket table.

        With offsets on the CPU the chunk is checked before any launch (ValueError) and the host's capacity bound advances by the
        longest sequence; offsets on the device are not read on the host (the bound advances by max_len), so a call with fixed
        (B, T, max_len) is CUDA-graph capturable after one eager call and can be replayed with new ids, timestamps and offsets."""
        self._check_extend_mode("extend_jagged")
        B = state.batch_size
        offsets, grow = self._check_jagged_chunk("extend_jagged", input_ids, offsets, max_len, timestamps, B, state.capacity,
                                                 "the state's capacity", top_k, num_candidates, exclude)
        if input_ids.device != state.lengths.device:
            raise ValueError(f"the state lives on {state.lengths.device}; got input_ids on {input_ids.device}")
        grow = int(grow.max()) if isinstance(grow, torch.Tensor) else grow
        return self._extend_state(state, input_ids, timestamps, offsets, max_len, grow, top_k, num_candidates, exclude)

    def _check_jagged_chunk(self, what: str, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int,
                            timestamps: Optional[torch.Tensor], B: int, limit: int, limit_name: str, top_k: Optional[int],
                            num_candidates: Optional[int], exclude: Optional[torch.Tensor]):
        """Argument check of a packed chunk of B sequences, all of it before the device is touched -> (offsets on the device, how
        far each sequence can grow its user: the lengths [B] for CPU offsets, max_len for device offsets)."""
        if isinstance(offsets, torch.Tensor) and offsets.dim() == 1 and offsets.numel() != B + 1:
            raise ValueError(f"{what}: offsets must be [{B + 1}] (one sequence per user of the call), got [{offsets.numel()}]")
        if isinstance(max_len, int) and max_len > limit:
            raise ValueError(f"{what}: max_len {max_len} exceeds {limit_name} ({limit})")
        self._check_serving_topk(what, top_k, num_candidates, exclude, B, input_ids.device)
        dev_offsets = self._check_jagged(what, input_ids, offsets, max_len, timestamps)
        return dev_offsets, (max_len if offsets.is_cuda else offsets[1:] - offsets[:-1])

    def _extend_state(self, state: HSTUState, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor], offsets: Optional[torch.Tensor],
                      max_len: int, grow: int, top_k: Optional[int], num_candidates: Optional[int], exclude: Optional[torch.Tensor]):
        """The body of ``extend`` (offsets None: a padded [B, max_len] chunk) and ``extend_jagged``, after their argument checks;
        ``grow`` advances the host's bound of every user's length."""
        if state.items_bound + grow > state.capacity:
            raise ValueError(f"extending by {grow} items could exceed the state's capacity ({state.items_bound} of {state.capacity} may be "
                             "used); start a new state with a larger capacity")
        use_time = self._check_cache_owner(state, timestamps, "state")
        ids = input_ids.contiguous()
        cache = state._struct()
        positions, last_row = Fn.hstu_cache_append(cache, ids, timestamps.contiguous() if timestamps is not None else None, offsets,
                                                   max_len)
        x = self._extend_blocks(ids, positions, cache, state.capacity, use_time, offsets=offsets, max_len=max_len)
        latest = x[self._last_tokens(last_row, offsets, max_len)]
        state.last_hidden.copy_(torch.where((last_row >= 0)[:, None], latest, state.last_hidden))
        state.items_bound += grow
        return self._hidden_select(state.last_hidden, top_k, num_candidates, exclude)

    @staticmethod
    def _last_tokens(last_row: torch.Tensor, offsets: Optional[torch.Tensor], n: int) -> torch.Tensor:
        """The token row of each user's last item (row 0 where the chunk had none): a packed chunk's append returns token rows, a
        padded one the row within the user's n slots."""
        tok = last_row.clamp(min=0).long()
        return tok if offsets is not None else tok + torch.arange(tok.numel(), device=tok.device) * n

    def _check_extend_mode(self, what: str) -> None:
        if self.precision == "fp32":
            raise RuntimeError(f"genrec_b200: {what} runs the bf16 path only; set_precision('bf16') or use last_logits")
        if self.training and any(isinstance(m, nn.Dropout) and m.p > 0 for m in self.modules()):
            raise RuntimeError(f"genrec_b200: {what} has no dropout; call model.eval()")

    def _check_cache_owner(self, cache, timestamps: Optional[torch.Tensor], what: str) -> bool:
        """Ties a state / pool to the parameter versions and the timestamp mode of its first write; returns the timestamp mode."""
        use_time = timestamps is not None and self.use_temporal_bias
        versions = tuple(p._version for p in self.parameters())
        if cache.param_versions is None:
            cache.param_versions, cache.has_time = versions, use_time
        elif cache.param_versions != versions:
            raise RuntimeError(f"genrec_b200: the model's parameters changed after this {what} was written; rebuild the {what}")
        elif cache.has_time != use_time:
            raise ValueError(f"timestamps must be given on every extend of a {what} or on none")
        return use_time

    def _extend_blocks(self, ids: torch.Tensor, positions: torch.Tensor, cache, capacity: int, use_time: bool,
                       users: Optional[torch.Tensor] = None, offsets: Optional[torch.Tensor] = None,
                       max_len: Optional[int] = None) -> torch.Tensor:
        """Embedding and every block of a chunk [B, n] (or, with ``offsets`` and ``max_len``, a packed chunk [T]) against ``cache`` (a
        dense HstuCache, or an HstuPool with ``users``) -> the final block's output [B * n or T, D] fp32, one row per token."""
        dev = ids.device
        # HSTU has no position table, so the embedding of a packed chunk is that of one [1, T] row
        x, _ = Fn.EmbedFn.apply(ids if offsets is None else ids.view(1, -1), self.item_embedding.weight, None, 1.0, 0, 0.0, 0, None, None)
        if offsets is not None:
            x = x.view(-1, self.embed_dim)
        if len(self.layers):
            rpb = self.layers[0].position_bias
            uniform, bucket0 = rpb.uniform_of(capacity, dev)
            pos_bucket = None if uniform else rpb.bucket_of_delta(capacity, dev)
            ntime = self.layers[0].temporal_bias.num_buckets if use_time else 0
            for i, layer in enumerate(self.layers):
                layer._bf16_provider = self._bf16_provider
                x = Fn.hstu_layer_extend(x, cache, i, positions, pos_bucket, bucket0, _thresholds_on(dev), layer.num_heads, rpb.num_buckets,
                                         ntime, layer._bf16_weights(), layer._params(), users=users, offsets=offsets, max_len=max_len)
        return x.view(-1, self.embed_dim)

    def _hidden_logits(self, hidden: torch.Tensor) -> torch.Tensor:
        return Fn.head_logits(hidden[:, None, :], self.final_norm.weight, self.final_norm.bias, self.item_embedding.weight,
                              self._table_mirror(), self.final_norm.eps)[:, 0, :]

    def new_pool(self, max_users: int, num_pages: int, page_size: int = 64, max_items: int = 2048) -> HSTUPool:
        """An empty paged cache for serving: ``num_pages`` pages of ``page_size`` items (a multiple of 64) shared by users
        0 .. max_users-1, each holding up to ``max_items`` (<= 16384) items, on the model's device."""
        return HSTUPool(max_users, num_pages, page_size, max_items, len(self.layers), self.embed_dim, self.item_embedding.weight.device)

    @torch.no_grad()
    def extend_users(self, pool: HSTUPool, users, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor] = None, *,
                     top_k: Optional[int] = None, num_candidates: Optional[int] = None, exclude: Optional[torch.Tensor] = None):
        """``extend`` for the users named by ``users`` [B] (int64, distinct, any subset of the pool's users in any order): append the
        non-zero ids of row b of ``input_ids`` [B, n] to the history of user ``users[b]`` in ``pool`` and return [B, V+1] fp32, row b
        being that user's next-item logits - what ``extend`` returns for the same user, i.e. ``last_logits`` of the left-padded
        concatenation of every item extended for them since their last ``pool.release``.  An all-pad row leaves its user untouched
        and returns their previous logits.  With ``top_k`` (1..64) it returns ``TopItems`` of the same rows instead (``exclude`` [B, E]
        int64: ids left out per row), selected without forming the logits; ``num_candidates`` (1..2048, not together with ``top_k``)
        returns up to 2048 of them, as ``retrieve`` does.

        With ``users`` on the CPU the call is refused before any launch if a user is out of range or repeated, or if the host
        bounds say a user could exceed ``max_items`` or the pool could run out of pages.  With ``users`` on the device (CUDA graphs)
        those checks are skipped: a row whose user is out of range or repeats an earlier row's counts as all padding (its logits are
        the head of a zero vector) and sets ``pool.errors()``, and items beyond ``max_items`` or without a free page are dropped in
        row order and flag their user in ``pool.overflowed()``."""
        self._check_extend_mode("extend_users")
        require_cuda(input_ids)
        ensure_device(input_ids.device)
        if input_ids.dim() != 2 or input_ids.device != pool.lengths.device:
            raise ValueError(f"input_ids must be [B, n] on {pool.lengths.device}; got {tuple(input_ids.shape)} on {input_ids.device}")
        B, n = input_ids.shape
        users = torch.as_tensor(users, dtype=torch.int64) if not isinstance(users, torch.Tensor) else users
        if users.shape != (B,):
            raise ValueError(f"users must have one entry per row of input_ids ({B}), got shape {tuple(users.shape)}")
        self._check_serving_topk("extend_users", top_k, num_candidates, exclude, B, input_ids.device)
        return self._extend_pool(pool, users, input_ids, timestamps, None, n, n, top_k, num_candidates, exclude)

    @torch.no_grad()
    def extend_users_jagged(self, pool: HSTUPool, users, input_ids: torch.Tensor, offsets: torch.Tensor, max_len: int,
                            timestamps: Optional[torch.Tensor] = None, *, top_k: Optional[int] = None,
                            num_candidates: Optional[int] = None, exclude: Optional[torch.Tensor] = None):
        """``extend_users`` on a packed chunk: sequence b (rows offsets[b] .. offsets[b+1]-1 of input_ids / timestamps [T], as in
        ``extend_jagged``) appends to user ``users[b]``, max_len <= the pool's max_items.  Returns what ``extend_users`` returns for
        the padded [B, max_len] chunk holding the same items per user, bit for bit, and leaves the pool (page tables, free pages,
        errors) as that call does, under the same device rules.

        With ``users`` on the CPU the call is refused before any launch as ``extend_users`` refuses it; the host's bound of each
        user advances by their exact length when the offsets are on the CPU too, and by max_len when the offsets are on the device
        (not read on the host).  With ``users`` on the device those checks are skipped.  A call with fixed (B, T, max_len) and
        device ``users`` / ``offsets`` is CUDA-graph capturable after one eager call."""
        self._check_extend_mode("extend_users_jagged")
        users = torch.as_tensor(users, dtype=torch.int64) if not isinstance(users, torch.Tensor) else users
        if users.dim() != 1:
            raise ValueError(f"users must be a 1-D tensor with one entry per sequence, got shape {tuple(users.shape)}")
        offsets, grow = self._check_jagged_chunk("extend_users_jagged", input_ids, offsets, max_len, timestamps, users.shape[0],
                                                 pool.max_items, "the pool's max_items", top_k, num_candidates, exclude)
        if input_ids.device != pool.lengths.device:
            raise ValueError(f"input_ids must be on {pool.lengths.device}; got {input_ids.device}")
        return self._extend_pool(pool, users, input_ids, timestamps, offsets, max_len, grow, top_k, num_candidates, exclude)

    def _extend_pool(self, pool: HSTUPool, users: torch.Tensor, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor],
                     offsets: Optional[torch.Tensor], max_len: int, grow, top_k: Optional[int], num_candidates: Optional[int],
                     exclude: Optional[torch.Tensor]):
        """The body of ``extend_users`` (offsets None: a padded [B, max_len] chunk) and ``extend_users_jagged``, after their argument
        checks; ``grow`` (an int or a [B] tensor) advances the host's bound of each CPU user's length."""
        dev = input_ids.device
        bound = None
        if not users.is_cuda:
            u_host = pool._host_users(users)
            bound = pool._check_room(u_host, grow)
        use_time = self._check_cache_owner(pool, timestamps, "pool")
        users = users.to(dev).long()
        ids = input_ids.contiguous()
        cache = pool._struct()
        positions, last_row, room = Fn.hstu_pool_append(cache, users, ids, timestamps.contiguous() if timestamps is not None else None,
                                                        offsets, max_len)
        x = self._extend_blocks(ids, positions, cache, pool.max_items, use_time, users=users, offsets=offsets, max_len=max_len)
        latest = x[self._last_tokens(last_row, offsets, max_len)]
        slot = torch.where(room >= 0, users, pool.max_users)     # rejected rows read and write the spare zero row
        hidden = torch.where((last_row >= 0)[:, None], latest, pool.last_hidden[slot])
        pool.last_hidden[slot] = hidden
        if bound is not None:
            pool.items_bound[u_host], pool.pages_bound = bound
        return self._hidden_select(hidden, top_k, num_candidates, exclude)

    @torch.no_grad()
    def evaluate_batch(self, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor], targets: torch.Tensor,
                       metrics: Optional[torch.Tensor] = None, *, exclude: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Leave-one-out metrics of one evaluation batch, accumulated ON THE DEVICE into ``metrics`` ([6] fp32: Recall@{1,5,10} hit
        counts, NDCG@{1,5,10} sums) - the loop of genrec/trainers/hstu_trainer.py:55-81 without per-sample ``.item()`` calls.
        Divide by the number of samples (and all-reduce across ranks) once at the end of the evaluation.

        At bf16 precision the target's rank is counted while the head scores the table (``Fn.head_rank_metrics``), so no
        [B, V+1] logits are formed and memory does not grow with the catalog; the ranks equal those of ``last_logits`` exactly.
        ``exclude`` ([B, E] int64, E <= 16384) leaves ids out of each row's ranking; a row whose target is excluded is not counted.
        At fp32 precision the metrics come from ``last_logits`` and ``exclude`` is refused."""
        if self.precision == "fp32":
            if exclude is not None:
                raise RuntimeError("genrec_b200: evaluate_batch with exclude runs the bf16 path only; set_precision('bf16')")
            return Fn.eval_rank_metrics(self.last_logits(input_ids, timestamps), targets, metrics)
        Fn.check_exclude_arg(exclude, input_ids.shape[0], input_ids.device)
        x = self.encode(input_ids, timestamps)
        return Fn.head_rank_metrics(x[:, -1, :], self.final_norm.weight, self.final_norm.bias, self._table_mirror(), self.final_norm.eps,
                                    targets, metrics, exclude)

    @torch.no_grad()
    def predict(self, input_ids: torch.Tensor, timestamps: Optional[torch.Tensor] = None, top_k: int = 10) -> torch.Tensor:
        """hstu.py:150-157."""
        logits, _ = self.forward(input_ids, timestamps)
        last_logits = logits[:, -1, :]
        last_logits[:, 0] = float("-inf")
        _, top_k_items = torch.topk(last_logits, top_k, dim=-1)
        return top_k_items
