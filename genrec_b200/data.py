"""Input contract of the hot path: collate functions (mirrors of genrec/data/amazon_hstu.py:137-200 and
genrec/data/amazon_sasrec.py:125-181), synthetic generators (SURVEY.md section 8d) and data-parallel batch sharding.
Host-side, pure Python/torch-CPU; nothing here computes model arithmetic.  ``sample_negatives`` draws the shared negatives of the
sampled-softmax head on whichever device its inputs live on."""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch


def hstu_collate_fn(batch: List[Dict], max_seq_len: int = 50):
    """LEFT-pad to the batch maximum (not max_seq_len), targets shifted by one, padded timestamps = 0
    (genrec/data/amazon_hstu.py:137-173)."""
    histories = [b["history"] for b in batch]
    stamps = [b["timestamps"] for b in batch]
    targets = [b["target"] for b in batch]
    max_len = min(max(len(h) for h in histories), max_seq_len)
    ids, tgs, tss = [], [], []
    for h, ts, t in zip(histories, stamps, targets):
        if len(h) > max_len:
            h, ts = h[-max_len:], ts[-max_len:]
        seq = list(h) + [t]
        ts_seq = list(ts) + [ts[-1] if ts else 0]
        pad = max_len + 1 - len(seq)
        seq, ts_seq = [0] * pad + seq, [0] * pad + ts_seq
        ids.append(seq[:-1]); tgs.append(seq[1:]); tss.append(ts_seq[:-1])
    return {"input_ids": torch.tensor(ids, dtype=torch.long), "targets": torch.tensor(tgs, dtype=torch.long),
            "timestamps": torch.tensor(tss, dtype=torch.long)}


def hstu_eval_collate_fn(batch: List[Dict], max_seq_len: int = 50):
    """genrec/data/amazon_hstu.py:176-200: targets is the single next item per sample."""
    histories = [b["history"] for b in batch]
    stamps = [b["timestamps"] for b in batch]
    max_len = min(max(len(h) for h in histories), max_seq_len)
    ids, tss = [], []
    for h, ts in zip(histories, stamps):
        if len(h) > max_len:
            h, ts = h[-max_len:], ts[-max_len:]
        pad = max_len - len(h)
        ids.append([0] * pad + list(h)); tss.append([0] * pad + list(ts))
    return {"input_ids": torch.tensor(ids, dtype=torch.long), "targets": torch.tensor([b["target"] for b in batch], dtype=torch.long),
            "timestamps": torch.tensor(tss, dtype=torch.long)}


def sasrec_collate_fn(batch: List[Dict], max_seq_len: int = 50):
    """genrec/data/amazon_sasrec.py:125-161 (same as the HSTU one without timestamps)."""
    out = hstu_collate_fn([dict(history=b["history"], timestamps=[0] * len(b["history"]), target=b["target"]) for b in batch], max_seq_len)
    return {"input_ids": out["input_ids"], "targets": out["targets"]}


def synthetic_batch(B: int, L: int, V: int, seed: int, full_length: bool = True):
    """SURVEY.md section 8(d): ids ~ Zipf(1.1) over 1..V, timestamps = 1.30e9 + cumsum(Exp(mean 3 days)); with
    full_length=False the lengths are ~U[L/4, L] and the batch is left-padded exactly like hstu_collate_fn."""
    g = torch.Generator().manual_seed(seed)
    w = torch.arange(1, V + 1, dtype=torch.float64).pow(-1.1)
    ids = torch.multinomial(w, B * (L + 1), replacement=True, generator=g).view(B, L + 1) + 1
    gaps = torch.empty(B, L).exponential_(1.0 / (3 * 86400.0), generator=g).long() + 1
    ts = 1_300_000_000 + torch.cumsum(gaps, 1)
    inp, tgt = ids[:, :L].clone(), ids[:, 1:].clone()
    if not full_length:
        lens = torch.randint(max(1, L // 4), L + 1, (B,), generator=g)
        for b in range(B):
            p = L - int(lens[b])
            inp[b, :p] = 0; ts[b, :p] = 0
            tgt[b, :max(p - 1, 0)] = 0
    return inp.contiguous(), ts.contiguous(), tgt.contiguous()


def shard_batch(batch: Dict[str, torch.Tensor], rank: int, world: int) -> Dict[str, torch.Tensor]:
    """Contiguous equal split of the global batch across data-parallel ranks (what Accelerate's prepared DataLoader does with
    split_batches=True; with the default split_batches=False every rank simply draws its own batch)."""
    out = {}
    for k, v in batch.items():
        n = v.shape[0]
        assert n % world == 0, "global batch must divide evenly across ranks"
        per = n // world
        out[k] = v[rank * per:(rank + 1) * per]
    return out


def collate_jagged(items: torch.Tensor, offsets: torch.Tensor, targets: torch.Tensor, max_seq_len: int = 50,
                   timestamps: "torch.Tensor | None" = None, max_len_in_batch: "int | None" = None) -> Dict[str, torch.Tensor]:
    """hstu_collate_fn / sasrec_collate_fn ON THE DEVICE: a jagged batch that already lives in HBM (items / timestamps [N] int64 in time
    order, offsets [B+1], one held-out target per user) -> the left-padded [B, L] batch dict, without a host round trip.
    L = min(longest history, max_seq_len); pass ``max_len_in_batch`` (the loader knows it) to avoid the one device sync that reading it
    from ``offsets`` costs."""
    from ._lib import GrbError, call, ptr, require_cuda
    require_cuda(items, offsets, targets)
    for t in (items, offsets, targets, timestamps):
        if t is not None and t.dtype != torch.int64:
            raise GrbError(f"genrec_b200 error -1: jagged batches are int64 (got {t.dtype})")
    B = offsets.numel() - 1
    if max_len_in_batch is None:
        max_len_in_batch = int((offsets[1:] - offsets[:-1]).max().item())
    L = max(1, min(int(max_len_in_batch), int(max_seq_len)))
    dev = items.device
    ids = torch.empty(B, L, dtype=torch.int64, device=dev)
    tgs = torch.empty(B, L, dtype=torch.int64, device=dev)
    tss = torch.empty(B, L, dtype=torch.int64, device=dev) if timestamps is not None else None
    call(dev, "grb_collate_jagged", ptr(items.contiguous()), ptr(timestamps.contiguous()) if timestamps is not None else None,
         ptr(offsets.contiguous()), ptr(targets.contiguous()), B, L, ptr(ids), ptr(tgs), ptr(tss))
    out = {"input_ids": ids, "targets": tgs}
    if tss is not None:
        out["timestamps"] = tss
    return out


def pack_jagged(items: torch.Tensor, offsets: torch.Tensor, targets: torch.Tensor, max_seq_len: int = 50,
                timestamps: "torch.Tensor | None" = None, num_tokens: "int | None" = None) -> Dict[str, torch.Tensor]:
    """``collate_jagged`` without the pads, for ``HSTU.forward_jagged`` and ``SASRec.forward_jagged``: the same jagged batch on the
    device (items / timestamps [N] int64 in time order, offsets [B+1], one held-out target per user) -> a packed batch.  Sequence b
    is hstu_collate_fn's row b with its pads removed: the last min(len_b, max_seq_len) items, the targets shifted by one with the
    held-out item last.  With ``timestamps=None`` that is sasrec_collate_fn's row b without its pads, SASRec's packed batch; its
    ``input_ids`` with the held-out targets [B] also serve ``evaluate_batch_jagged``.
    Returns input_ids, targets (and timestamps) [T], offsets [B+1] (sequence b = rows offsets[b] .. offsets[b+1]-1), the host int
    max_len and overflow (a 0-dim bool on the device).

    Without ``num_tokens`` T is the packed total and max_len the longest packed length, read from the device in one
    synchronisation.  With ``num_tokens`` T = num_tokens and max_len = max_seq_len, with no synchronisation (a captured step keeps
    fixed shapes): rows past the packed total are idle (id 0, target 0, timestamp 0), and a batch that does not fit sets
    ``overflow``, is cut at T and writes nothing past it - do not train on it."""
    from ._lib import GrbError, call, ptr, require_cuda
    require_cuda(items, offsets, targets)
    for t in (items, offsets, targets, timestamps):
        if t is not None and t.dtype != torch.int64:
            raise GrbError(f"genrec_b200 error -1: jagged batches are int64 (got {t.dtype})")
    B = offsets.numel() - 1
    if B < 1 or int(max_seq_len) < 1:
        raise ValueError(f"pack_jagged needs B >= 1 and max_seq_len >= 1 (got {B}, {max_seq_len})")
    if num_tokens is None:
        lens = (offsets[1:] - offsets[:-1]).clamp(0, int(max_seq_len))
        total, longest = torch.stack([lens.sum(), lens.max()]).tolist()
        T, max_len = max(1, int(total)), max(1, int(longest))
    else:
        if int(num_tokens) < 1:
            raise ValueError(f"num_tokens must be positive, got {num_tokens}")
        T, max_len = int(num_tokens), int(max_seq_len)
    dev = items.device
    ids = torch.empty(T, dtype=torch.int64, device=dev)
    tgs = torch.empty(T, dtype=torch.int64, device=dev)
    tss = torch.empty(T, dtype=torch.int64, device=dev) if timestamps is not None else None
    out_off = torch.empty(B + 1, dtype=torch.int64, device=dev)
    info = torch.empty(2, dtype=torch.int64, device=dev)
    call(dev, "grb_pack_jagged", ptr(items.contiguous()), ptr(timestamps.contiguous()) if timestamps is not None else None,
         ptr(offsets.contiguous()), ptr(targets.contiguous()), B, int(max_seq_len), T, ptr(ids), ptr(tgs), ptr(tss), ptr(out_off), ptr(info))
    out = {"input_ids": ids, "targets": tgs, "offsets": out_off, "max_len": max_len, "overflow": info[0] > T}
    if tss is not None:
        out["timestamps"] = tss
    return out


def pack_tiger(user_ids: torch.Tensor, item_tokens: torch.Tensor, token_offsets: torch.Tensor, target_ids: torch.Tensor, max_items: int = 20,
               num_tokens: "int | None" = None) -> Dict[str, torch.Tensor]:
    """TIGER's ``pad_collate`` (genrec/trainers/tiger_trainer.py:27-80) without the pads, for ``Tiger.forward_jagged`` and
    ``generate_jagged``: user b's semantic-id tokens are item_tokens[token_offsets[b] : token_offsets[b+1]] (three per item, in the
    reference's order; int64), user_ids [B], target_ids [B, S].  Sequence b of the packed encoder memory is its user row followed by
    its last min(n_b, 3 max_items) item tokens: pad_collate's row b (with the user token in front, as Tiger.forward puts it) without
    its pads.  Returns user_input_ids [B], item_input_ids and token_type_ids [T] (types arange(n) % 3; the user row holds id 0, type
    0, and forward_jagged puts the user embedding there), mem_offsets [B+1], the host int max_len, target_input_ids and
    target_token_type_ids [B, S] (types arange(S)), and overflow (a 0-dim bool).  Every tensor lives on item_tokens' device.

    Without ``num_tokens`` T is the packed total and max_len the longest sequence, read in one synchronisation.  With ``num_tokens``
    T = num_tokens and max_len = 1 + 3 max_items, with no synchronisation (a captured call keeps fixed shapes): rows past the packed
    total are idle, and a batch that does not fit sets ``overflow`` and is cut at T - do not use it."""
    dev = item_tokens.device
    for t in (user_ids, item_tokens, token_offsets, target_ids):
        if t.dtype != torch.int64:
            raise ValueError(f"pack_tiger: every input is int64 (got {t.dtype})")
    if token_offsets.dim() != 1 or token_offsets.numel() < 2 or user_ids.numel() != token_offsets.numel() - 1:
        raise ValueError("pack_tiger: token_offsets must be [B+1] with B >= 1 and user_ids [B]")
    if target_ids.dim() != 2 or target_ids.shape[0] != user_ids.numel():
        raise ValueError(f"pack_tiger: target_ids must be [B, S], got {tuple(target_ids.shape)}")
    if int(max_items) < 1:
        raise ValueError(f"pack_tiger: max_items must be positive, got {max_items}")
    off = token_offsets.to(dev)
    B, cap = off.numel() - 1, 3 * int(max_items)
    lens = (off[1:] - off[:-1]).clamp(0, cap)
    start = off[1:] - lens                                     # the last min(n_b, cap) tokens
    mem_off = torch.zeros(B + 1, dtype=torch.int64, device=dev)
    mem_off[1:] = torch.cumsum(lens + 1, 0)
    if num_tokens is None:
        total, longest = torch.stack([mem_off[-1], lens.max() + 1]).tolist()
        T, max_len = int(total), int(longest)
    else:
        if int(num_tokens) < 1:
            raise ValueError(f"num_tokens must be positive, got {num_tokens}")
        T, max_len = int(num_tokens), 1 + cap
    rows = torch.arange(T, dtype=torch.int64, device=dev)
    b = torch.searchsorted(mem_off[1:], rows, right=True)      # sequence of each row; B for idle rows
    bc = b.clamp(max=B - 1)
    k = rows - mem_off[bc]                                     # 0 = the user row
    item = (b < B) & (k > 0)
    if item_tokens.numel():
        tok = (start[bc] + k - 1).clamp(0, item_tokens.numel() - 1)
        ids = torch.where(item, item_tokens[tok], torch.zeros_like(rows))
    else:
        ids = torch.zeros_like(rows)
    types = torch.where(item, (k - 1) % 3, torch.zeros_like(rows))
    S = target_ids.shape[1]
    return {"user_input_ids": user_ids.reshape(-1).to(dev), "item_input_ids": ids, "token_type_ids": types,
            "mem_offsets": mem_off.clamp(max=T), "max_len": max_len, "target_input_ids": target_ids.to(dev),
            "target_token_type_ids": torch.arange(S, dtype=torch.int64, device=dev).unsqueeze(0).expand(B, S).contiguous(),
            "overflow": mem_off[-1] > T}


def sample_negatives(num_items: int, n: int, *, probs: Optional[torch.Tensor] = None, generator: Optional[torch.Generator] = None,
                     device=None) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """The shared negatives of one sampled-softmax step: ``(negatives [n] int64 in 1..num_items, log_q [num_items + 1] fp32 | None)``,
    drawn with replacement, on the device and without a host synchronisation (so a captured step can redraw them).

    Without ``probs`` the draw is uniform and ``log_q`` is None (a constant correction changes nothing).  ``probs`` [num_items + 1]
    are non-negative item frequencies or probabilities (entry 0, the padding id, is never drawn): the draw is
    ``torch.multinomial(probs[1:], n, replacement=True)`` and ``log_q = log(probs / probs[1:].sum())`` (``-inf`` for never-drawn
    items; such an item only ever appears as a target, where a finite correction is needed, so pass smoothed frequencies)."""
    if num_items < 1 or n < 1:
        raise ValueError(f"sample_negatives needs num_items >= 1 and n >= 1 (got {num_items}, {n})")
    if probs is None:
        dev = device if device is not None else (generator.device if generator is not None else "cpu")
        return torch.randint(1, num_items + 1, (n,), dtype=torch.int64, device=dev, generator=generator), None
    if tuple(probs.shape) != (num_items + 1,):
        raise ValueError(f"probs must be [{num_items + 1}] (one entry per id 0..num_items), got {tuple(probs.shape)}")
    w = probs.detach().float()
    negatives = torch.multinomial(w[1:], n, replacement=True, generator=generator) + 1
    log_q = torch.log(w / w[1:].sum())
    return negatives, log_q
