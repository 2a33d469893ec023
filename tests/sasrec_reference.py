"""fp64 restatement of the SASRec training step (genrec/models/sasrec.py:79-130, :152-165, :192-266; oracle/sasrec.py without
dropout) in plain torch, with every dropout taken as an explicit keep-scale tensor, and the helper that restates the dropout masks
the kernels of genrec_b200.sasrec draw from (seed, site, row key).

A mask is a keep-scale tensor: 0 where dropped, the keep scale elsewhere.  The kernels' scale is attention_reference.keep_scale(p)
(2^16 / (2^16 - round(p 2^16)) in fp32), not torch's 1 / (1 - p).  The row-wise masks are over the T token rows (T = B L for a
padded batch, flattened row-major):

  "emb"   [T, D]                 emb_dropout after the embedding and position sum           sasrec.py:110
  per block l, in lists of num_blocks:
  "attn"  [B, H, L, L]           the attention probabilities, after the query mask          sasrec.py:236
          packed: one [1, H, n, n] per sequence (n its length)
  "hid"   [T, ffn]               the FFN dropout after ReLU                                 sasrec.py:264
  "out"   [T, D]                 the FFN dropout on fc2's output                            sasrec.py:265

The packed form (`forward` with `packed`, the layout of data.pack_jagged) takes input_ids / targets [T] and offsets (sequence b =
rows offsets[b] .. offsets[b+1] - 1).  Item i of a sequence of length n sits at position P - n + i, P the batch's longest sequence,
as in sasrec_collate_fn's left-padded batch; each sequence attends to itself alone; rows outside every sequence are idle: x = 0,
target 0.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from tests import dense_reference as dr
from tests.attention_reference import attn_keep, drop_mask, keep_scale, sas_site
from tests.hstu_block_reference import effective_seed

EPS = 1e-8                                  # every LayerNorm of SASRec (sasrec.py:59, :150-151)
SITE_HID, SITE_OUT = 1, 2                   # genrec_b200.sasrec: site 8 layer + which; the attention core's is sas_site(layer)


def _drop(x, mask):
    if mask is None:
        return x
    if tuple(mask.shape) != tuple(x.shape):
        raise ValueError(f"dropout mask {tuple(mask.shape)} for a tensor {tuple(x.shape)}")
    return x * mask.to(device=x.device, dtype=x.dtype)


def _ln(prm, name, x):
    return F.layer_norm(x, (x.shape[-1],), prm[name + ".weight"], prm[name + ".bias"], EPS)


def _attention(Q, K, V, valid, H, keep):
    """MultiHeadAttention.forward after the projections (sasrec.py:205-240): Q, K, V [b, n, D], valid [b, n] (1 = a real item)."""
    b, n, D = Q.shape
    dh = D // H
    heads = lambda t: t.reshape(b, n, H, dh).transpose(1, 2)
    q, k, v = heads(Q), heads(K), heads(V)
    scores = (q @ k.transpose(-2, -1)) * dh ** -0.5
    scores = scores.masked_fill(~valid[:, None, None, :], -1e9)
    causal = torch.triu(torch.ones(n, n, dtype=torch.bool, device=Q.device), diagonal=1)
    scores = scores.masked_fill(causal[None, None], -1e9)
    a = F.softmax(scores, dim=-1) * valid[:, None, :, None].to(scores.dtype)
    a = _drop(a, keep)
    return (a @ v).transpose(1, 2).reshape(b, n, D)


def _block(prm, pre, x, valid, H, keep, hid, out, offsets):
    """SASRecBlock.forward and the trailing `x * mask` (sasrec.py:116, :152-165) on x [T, D]; valid [T] bool.  offsets None: x is
    a padded batch [B, L] flattened; otherwise each sequence attends alone and the idle rows take no attention output."""
    q = _ln(prm, pre + "norm1", x)
    Q = F.linear(q, prm[pre + "attention.q_proj.weight"], prm[pre + "attention.q_proj.bias"])     # Q from LN1(x)
    K = F.linear(x, prm[pre + "attention.k_proj.weight"], prm[pre + "attention.k_proj.bias"])     # K and V from x
    V = F.linear(x, prm[pre + "attention.v_proj.weight"], prm[pre + "attention.v_proj.bias"])
    if offsets is None:
        B, L = valid.shape
        att = _attention(Q.view(B, L, -1), K.view(B, L, -1), V.view(B, L, -1), valid, H, keep).reshape(B * L, -1)
        rowmask = valid.reshape(-1)
    else:
        parts = [Q[:offsets[0]] * 0]
        for s, (r0, r1) in enumerate(zip(offsets, offsets[1:])):
            sl = slice(r0, r1)
            parts.append(_attention(Q[sl][None], K[sl][None], V[sl][None], valid[sl][None], H,
                                    None if keep is None else keep[s])[0])
        parts.append(Q[offsets[-1]:] * 0)
        att = torch.cat(parts)
        rowmask = valid
    h = att + q                                                                                   # residual = the normalised query
    f = _drop(F.relu(F.linear(_ln(prm, pre + "norm2", h), prm[pre + "ffn.fc1.weight"], prm[pre + "ffn.fc1.bias"])), hid)
    y = _drop(F.linear(f, prm[pre + "ffn.fc2.weight"], prm[pre + "ffn.fc2.bias"]), out) + h
    return y * rowmask[:, None].to(y.dtype)


def seeded_params(cfg, seed):
    """SASRec's state_dict (cfg: SASRec's constructor arguments by name) drawn at the scale of its initialisation, with the norm
    gains and every bias drawn away from 1 and 0 so that a swapped or skipped one shows; row 0 of the item table is zero."""
    V, P, D, ffn = cfg["num_items"] + 1, cfg["max_seq_len"], cfg["embed_dim"], cfg["ffn_dim"]
    g = torch.Generator().manual_seed(seed)
    rnd = lambda *shape, scale: scale * torch.randn(*shape, generator=g)
    prm = {"item_embedding.weight": rnd(V, D, scale=(2.0 / (V + D)) ** 0.5), "position_embedding.weight": rnd(P, D, scale=(2.0 / (P + D)) ** 0.5)}
    prm["item_embedding.weight"][0] = 0
    for l in range(cfg["num_blocks"]):
        pre = f"blocks.{l}."
        for name in ("q_proj", "k_proj", "v_proj"):
            prm[pre + f"attention.{name}.weight"] = rnd(D, D, scale=D ** -0.5)
            prm[pre + f"attention.{name}.bias"] = rnd(D, scale=0.1)
        prm[pre + "ffn.fc1.weight"], prm[pre + "ffn.fc1.bias"] = rnd(ffn, D, scale=D ** -0.5), rnd(ffn, scale=0.1)
        prm[pre + "ffn.fc2.weight"], prm[pre + "ffn.fc2.bias"] = rnd(D, ffn, scale=ffn ** -0.5), rnd(D, scale=0.1)
        for n in ("norm1", "norm2"):
            prm[pre + n + ".weight"], prm[pre + n + ".bias"] = 1 + rnd(D, scale=0.1), rnd(D, scale=0.1)
    prm["final_norm.weight"], prm["final_norm.bias"] = 1 + rnd(D, scale=0.1), rnd(D, scale=0.1)
    return prm


def positions(offsets, T):
    """the packed position of each of the T rows (-1 on idle rows) and P: item i of a sequence of length n at P - n + i"""
    P = max([b - a for a, b in zip(offsets, offsets[1:])] + [0])
    pos = [-1] * T
    for a, b in zip(offsets, offsets[1:]):
        for i in range(b - a):
            pos[a + i] = P - (b - a) + i
    return torch.tensor(pos), P


def forward(prm, cfg, batch, masks=None, packed=False):
    """-> (logits [B, L, V+1] | [T, V+1], loss).  prm: SASRec's state_dict names; cfg: num_heads, num_blocks; batch: input_ids
    and targets ([B, L], or [T] with offsets when packed); masks: the dict of the module docstring, or None (no dropout)."""
    H, nb = cfg["num_heads"], cfg["num_blocks"]
    E = prm["item_embedding.weight"]
    D = E.shape[1]
    ids, tg = batch["input_ids"], batch["targets"]
    m = masks or {}
    pick = lambda k, l: m[k][l] if k in m else None
    if packed:
        offsets = [int(o) for o in batch["offsets"]]
        T = ids.numel()
        pos, _ = positions(offsets, T)
        pos = pos.to(ids.device)
        valid = (ids.reshape(-1) != 0) & (pos >= 0)
        pe = prm["position_embedding.weight"][pos.clamp(min=0)]
    else:
        offsets = None
        B, L = ids.shape
        T = B * L
        valid = ids != 0
        pe = prm["position_embedding.weight"][:L].repeat(B, 1)
    x = F.embedding(ids.reshape(-1), E, padding_idx=0) * (D ** 0.5) + pe                  # sasrec.py:103-107
    x = _drop(x, m.get("emb")) * valid.reshape(-1, 1).to(x.dtype)                         # :110-111
    for l in range(nb):
        x = _block(prm, f"blocks.{l}.", x, valid, H, pick("attn", l), pick("hid", l), pick("out", l), offsets)
    x = _ln(prm, "final_norm", x)
    logits = x @ E.T                                                                      # :121
    loss = F.cross_entropy(logits, tg.reshape(-1), ignore_index=0)                        # :126-128
    return (logits if packed else logits.view(B, L, -1)), loss


def step(params, cfg, batch, masks=None, packed=False, dtype=torch.float64, device=None, autocast=False):
    """Forward and backward: -> {"logits", "loss", "grads": {name: gradient}}.  dtype / autocast: the same step in fp32 under bf16
    torch.autocast is the yardstick of the kernels' error."""
    device = device or next(iter(params.values())).device
    prm = {k: v.detach().to(device=device, dtype=dtype).requires_grad_(True) for k, v in params.items()}
    b = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}
    with torch.autocast(torch.device(device).type, dtype=torch.bfloat16, enabled=autocast):
        logits, loss = forward(prm, cfg, b, masks, packed)
    loss.backward()
    return {"logits": logits.detach(), "loss": loss.detach(), "grads": {k: v.grad for k, v in prm.items() if v.grad is not None}}


# ------------------------------------------------------------------------------------------------ the kernels' masks
def packed_attn_keep(tok0, n, H, p, seed, site, device="cpu"):
    """[1, H, n, n] keep-scale matrix of the packed core: query i of the sequence starting at token row tok0, head h, key j has
    row key (tok0 + i) H + h (mod 2^32) and column j."""
    rows = (tok0 + np.arange(n, dtype=np.int64))[None, :] * H + np.arange(H, dtype=np.int64)[:, None]
    drop = drop_mask(rows.reshape(-1) & 0xFFFFFFFF, n, p, seed, site)
    return torch.from_numpy(np.where(drop, 0.0, keep_scale(p)[1])).view(1, H, n, n).to(device)


def kernel_step_masks(cfg, p, seed, seed_dev_value, shape, device="cpu"):
    """Every mask one SASRec.forward / forward_jagged step draws, as the kernels draw it: the effective seed (seed + *seed_dev), the
    embedding at site 250, block l's attention core at 8 l + 3 and its FFN at 8 l + 1 / 8 l + 2; row-wise masks keyed by token
    row, the padded core by (b H + h) L + i, the packed core by (tok0 + i) H + h.  cfg: embed_dim, num_heads, ffn_dim,
    num_blocks; shape: ("padded", B, L) or ("packed", T, offsets)."""
    D, H, ffn, nb = cfg["embed_dim"], cfg["num_heads"], cfg["ffn_dim"], cfg["num_blocks"]
    s = effective_seed(seed, p, seed_dev_value)
    T = shape[1] * shape[2] if shape[0] == "padded" else shape[1]
    rows = range(T)
    out = {"emb": dr.keep(rows, D, p, s, dr.SITE_EMBED, device), "attn": [], "hid": [], "out": []}
    for l in range(nb):
        if shape[0] == "padded":
            out["attn"].append(attn_keep(shape[1], H, shape[2], shape[2], p, s, sas_site(l), device))
        else:
            offs = [int(o) for o in shape[2]]
            out["attn"].append([packed_attn_keep(a, b - a, H, p, s, sas_site(l), device) for a, b in zip(offs, offs[1:])])
        out["hid"].append(dr.keep(rows, ffn, p, s, 8 * l + SITE_HID, device))
        out["out"].append(dr.keep(rows, D, p, s, 8 * l + SITE_OUT, device))
    return out


def mask_sources(masks):
    """(name, tensor) of every mask a step draws, for checks that each drops something"""
    yield "emb", masks["emb"]
    for l in range(len(masks["hid"])):
        a = masks["attn"][l]
        yield f"attn {l}", torch.cat([t.reshape(-1) for t in a]) if isinstance(a, list) else a
        yield f"hid {l}", masks["hid"][l]
        yield f"out {l}", masks["out"][l]


def ones_masks(cfg, shape, device="cpu"):
    """a step's masks at p = 0: every entry 1"""
    return kernel_step_masks(cfg, 0.0, 0, None, shape, device)
