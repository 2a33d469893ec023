"""fp64 restatement of the TIGER training step (genrec/models/tiger.py:150-246 with genrec/modules/transformer.py and
genrec/modules/normalize.py) in plain torch, with every dropout taken as an explicit keep-scale tensor, and the helpers that restate
the dropout masks the kernels of genrec_b200.tiger draw from (seed, site).

A mask is a keep-scale tensor shaped like the tensor it multiplies: 0 where dropped, the keep scale elsewhere.  The kernels' scale is
attention_reference.keep_scale(p) (2^16 / (2^16 - round(p 2^16)) in fp32), not torch's 1 / (1 - p).  `step` consumes the masks in
the reference's call order (masks=None: no dropout):

  Tiger.drop on norm_context(encoder input) [B, 1+N, E]                tiger.py:191
  Tiger.drop on norm(decoder input) [B, S+1, E]                        tiger.py:192
  per encoder block                                                     transformer.py:303-323
    attention probabilities [B, H, L, L]                                transformer.py:153-154
    dropout1 on the self-attention branch [B, L, D]
    the FFN hidden dropout [B, L, 1024]                                 transformer.py:185-188
    dropout2 on the FFN branch [B, L, D]
  per decoder block: self-attention probabilities [B, H, S+1, S+1], dropout1, cross-attention probabilities [B, H, S+1, 1+N],
    dropout_cross [B, S+1, D], the FFN hidden dropout, dropout2.

The packed form (`step` with `packed`, the layout of data.pack_tiger) takes the encoder's row-wise masks over the T packed rows
([T, E], [T, D], [T, 1024]), the encoder self-attention masks as [T, H, max_len] (row t, head h, key j of t's sequence: the packed
core keys its dropout by token row, t H + h) and the cross-attention masks as [B, H, S+1, max_len].  Each user's memory runs through
the attention alone; rows past offsets[B] are idle and reach nothing.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from tests import dense_reference as dr
from tests.attention_reference import attn_keep, drop_mask, keep_scale

EPS = 1e-6                  # RMSNorm / RootMeanSquareLayerNorm (normalize.py:42, :77)
FFN_DIM = 1024              # tiger.py:140
NUM_BUCKETS, MAX_DISTANCE = 32, 128   # transformer.py:225-227


# ------------------------------------------------------------------------------------------------ the step
def _drop(x, mask):
    if mask is None:
        return x
    if tuple(mask.shape) != tuple(x.shape):
        raise ValueError(f"dropout mask {tuple(mask.shape)} for a tensor {tuple(x.shape)}")
    return x * mask.to(device=x.device, dtype=x.dtype)


def _rms(x, w):
    """normalize.py:47-55 and :85-96 (the same value: x rsqrt(mean(x^2) + eps) w)"""
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + EPS) * w


def _buckets(q_len, k_len, device):
    """transformer.py:13-41 at (32, 128, bidirectional): [q_len, k_len] bucket of memory position j - context position i"""
    rp = torch.arange(k_len, device=device)[None, :] - torch.arange(q_len, device=device)[:, None]
    n = -rp
    half = NUM_BUCKETS // 2
    sign = (n < 0).long()
    n = n.abs()
    exact = half // 2
    large = exact + (torch.log(n.float() / exact + 1e-6) / math.log(MAX_DISTANCE / exact) * (half - exact)).long().clamp(max=half - exact - 1)
    return torch.where(n < exact, n, large) + sign * half


def _attention(prm, pre, xq, xkv, H, key_pad, causal, mask):
    """T5Attention.forward (transformer.py:119-159) on xq [b, Lq, D] and, for cross-attention, xkv [b, Lk, D]"""
    D = xq.shape[-1]
    dh = D // H
    cross = xkv is not None
    if cross:
        k, v = F.linear(xkv, prm[pre + "k.weight"]), F.linear(xkv, prm[pre + "v.weight"])
    else:
        k, v = F.linear(xq, prm[pre + "kv.weight"]).chunk(2, dim=-1)
    q = F.linear(xq, prm[pre + "q.weight"])
    heads = lambda t: t.reshape(t.shape[0], t.shape[1], H, dh).transpose(1, 2)
    q, k, v = heads(q), heads(k), heads(v)
    scores = torch.matmul(q, k.transpose(-2, -1)) * (1.0 / math.sqrt(dh))
    Lq, Lk = q.shape[-2], k.shape[-2]
    if not cross:                                            # the relative-position bias (transformer.py:84-104, :138-141)
        idx = _buckets(Lq, Lk, xq.device)[None] + (torch.arange(H, device=xq.device) * NUM_BUCKETS)[:, None, None]
        scores = scores + F.embedding(idx, prm[pre + "rel_bias.weight"])[..., 0][None]
    if key_pad is not None:
        scores = scores.masked_fill(key_pad[:, None, None, :], -1e9)
    if causal:
        scores = scores + torch.triu(torch.full((Lq, Lk), float("-inf"), device=xq.device), diagonal=1).to(scores.dtype)
    attn = _drop(torch.softmax(scores, dim=-1), mask)
    out = torch.matmul(attn, v).transpose(1, 2).reshape(xq.shape[0], Lq, D)
    return F.linear(out, prm[pre + "o.weight"])


def _ffn(prm, pre, x, masks):
    """x + dropout2(wo(dropout(relu(wi(norm2(x)))))) (transformer.py:181-189, :323)"""
    h = _drop(F.relu(F.linear(_rms(x, prm[pre + "norm2.weight"]), prm[pre + "ff.wi.weight"])), next(masks))
    return x + _drop(F.linear(h, prm[pre + "ff.wo.weight"]), next(masks))


class _Masks:
    """the masks in call order; None for every call when there are none"""

    def __init__(self, masks):
        self.it = iter(masks) if masks is not None else None

    def __next__(self):
        if self.it is None:
            return None
        m = next(self.it, None)
        if m is None:
            raise ValueError("fewer dropout masks than dropout calls")
        return m

    def done(self):
        if self.it is not None and next(self.it, None) is not None:
            raise ValueError("more dropout masks than dropout calls")


def _per_user(offsets, fn):
    """fn(b, r0, r1) over the users of a packed batch"""
    return [fn(b, offsets[b], offsets[b + 1]) for b in range(len(offsets) - 1)]


def _encoder(prm, cfg, x, key_pad, masks, offsets=None):
    H = cfg["num_heads"]
    for l in range(cfg["n_layers"] // 2):
        pre = f"transformer.encoder.layers.{l}."
        xn = _rms(x, prm[pre + "norm1.weight"])
        a_mask = next(masks)
        if offsets is None:
            a = _attention(prm, pre + "self_attn.attn.", xn, None, H, key_pad, False, a_mask)
        else:                                                # each user's rows alone; idle rows take no attention output
            a = torch.cat([xn[:offsets[0]] * 0] + _per_user(offsets, lambda b, r0, r1: _attention(
                prm, pre + "self_attn.attn.", xn[r0:r1][None], None, H, None, False,
                None if a_mask is None else a_mask[r0:r1, :, :r1 - r0].transpose(0, 1)[None])[0]) + [xn[offsets[-1]:] * 0])
        x = _ffn(prm, pre, x + _drop(a, next(masks)), masks)
    return x


def _decoder(prm, cfg, x, memory, memory_pad, masks, offsets=None):
    H = cfg["num_heads"]
    for l in range(cfg["n_layers"] // 2):
        pre = f"transformer.decoder.layers.{l}."
        a = _attention(prm, pre + "self_attn.attn.", _rms(x, prm[pre + "norm1.weight"]), None, H, None, True, next(masks))
        x = x + _drop(a, next(masks))
        xn, c_mask = _rms(x, prm[pre + "norm_cross.weight"]), next(masks)
        if offsets is None:
            c = _attention(prm, pre + "cross_attn.attn.", xn, memory, H, memory_pad, False, c_mask)
        else:
            c = torch.cat(_per_user(offsets, lambda b, r0, r1: _attention(
                prm, pre + "cross_attn.attn.", xn[b:b + 1], memory[r0:r1][None], H, None, False,
                None if c_mask is None else c_mask[b:b + 1, :, :, :r1 - r0])))
        x = _ffn(prm, pre, x + _drop(c, next(masks)), masks)
    return x


def _sem(prm, cfg, ids, types):
    """SemIdEmbedding (embedding.py:42-43), padding row without a gradient"""
    w = prm["sem_id_embedding.emb.weight"]
    return F.embedding(types * cfg["num_item_embeddings"] + ids, w, padding_idx=w.shape[0] - 1)


def forward(prm, cfg, batch, masks=None, packed=False):
    """-> (logits [B, S+1, V], loss).  prm: the state_dict names of Tiger; batch: Tiger.forward's arguments by name (packed:
    forward_jagged's, mem_offsets on any device).  masks: keep-scale tensors in call order (module docstring) or None."""
    mk = _Masks(masks)
    users = batch["user_input_ids"].reshape(-1)
    B = users.numel()
    user_emb = F.embedding(users % cfg["num_user_embeddings"], prm["user_id_embedding.emb.weight"])   # embedding.py:73-74
    tgt, tgt_t = batch["target_input_ids"], batch["target_token_type_ids"]
    dec_in = torch.cat([prm["bos_embedding"].repeat(B, 1, 1), _sem(prm, cfg, tgt, tgt_t)], dim=1)         # tiger.py:176-179
    if not packed:
        enc_in = torch.cat([user_emb[:, None], _sem(prm, cfg, batch["item_input_ids"], batch["token_type_ids"])], dim=1)   # :166-173
        pad = torch.cat([torch.zeros(B, 1, dtype=torch.bool, device=users.device), batch["seq_mask"] == 0], dim=1)     # :183-189
        offsets = None
    else:                                                    # row offsets[b] is user b's row
        offsets = batch["mem_offsets"].tolist()
        enc_in = _sem(prm, cfg, batch["item_input_ids"], batch["token_type_ids"])
        enc_in = enc_in.index_copy(0, torch.tensor(offsets[:-1], device=enc_in.device), user_emb)
        pad = None
    enc_in = F.linear(_drop(_rms(enc_in, prm["norm_context.weight"]), next(mk)), prm["in_proj_context.weight"])   # :191
    dec_in = F.linear(_drop(_rms(dec_in, prm["norm.weight"]), next(mk)), prm["in_proj.weight"])                   # :192
    memory = _encoder(prm, cfg, enc_in, pad, mk, offsets)
    out = _decoder(prm, cfg, dec_in, memory, pad, mk, offsets)
    mk.done()
    logits = F.linear(out, prm["output_head.weight"])                                                         # :207
    target = tgt_t * cfg["num_item_embeddings"] + tgt                                                          # :232-240
    ll = logits[:, :-1, :]
    loss = F.cross_entropy(ll.reshape(-1, ll.size(-1)), target.reshape(-1), reduction="none").reshape(B, -1).sum(dim=1).mean()
    return logits, loss


def step(params, cfg, batch, masks=None, packed=False, dtype=torch.float64, device=None, autocast=False):
    """Forward and backward: -> {"logits", "loss", "grads": {name: gradient}} (parameters without a gradient left out).  dtype /
    autocast: the same step in fp32 under bf16 torch.autocast is the yardstick of the kernels' error."""
    device = device or next(iter(params.values())).device
    prm = {k: v.detach().to(device=device, dtype=dtype).requires_grad_(True) for k, v in params.items()}
    b = {k: (v.to(device) if isinstance(v, torch.Tensor) else v) for k, v in batch.items()}
    with torch.autocast(torch.device(device).type, dtype=torch.bfloat16, enabled=autocast):
        logits, loss = forward(prm, cfg, b, masks, packed)
    loss.backward()
    return {"logits": logits.detach(), "loss": loss.detach(), "grads": {k: v.grad for k, v in prm.items() if v.grad is not None}}


# ------------------------------------------------------------------------------------------------ the kernels' masks
def keep_tensor(drop, p):
    """keep-scale tensor of a bool drop mask (True = dropped) at the kernels' scale"""
    return torch.where(torch.as_tensor(drop), 0.0, keep_scale(p)[1]).double()


def ffn_masks(lead_shape, D, p, seed, site, device="cpu"):
    """_FfnFn's epilogue masks over its rows flattened: the hidden mask at `site` [*lead, 1024], the output mask at site + 1 [*lead, D]"""
    rows = range(int(np.prod(lead_shape)))
    return (dr.keep(rows, FFN_DIM, p, seed, site, device).view(*lead_shape, FFN_DIM),
            dr.keep(rows, D, p, seed, site + 1, device).view(*lead_shape, D))


def attn_mask_padded(B, H, Lq, Lk, p, seed, site, device="cpu"):
    """the T5 core on a padded batch: row key (b H + h) Lq + i, column j -> [B, H, Lq, Lk]"""
    return attn_keep(B, H, Lq, Lk, p, seed, site, device)


def attn_mask_packed_self(T, H, max_len, p, seed, site, device="cpu"):
    """the packed self-attention core: row key t H + h of token row t, column j -> [T, H, max_len]"""
    return keep_tensor(drop_mask(np.arange(T * H), max_len, p, seed, site), p).view(T, H, max_len).to(device)


def attn_mask_packed_cross(B, H, Lq, max_len, p, seed, site, device="cpu"):
    """the packed cross-attention core: the dense queries keep the padded keys (b H + h) Lq + i -> [B, H, Lq, max_len]"""
    return attn_keep(B, H, Lq, max_len, p, seed, site, device)


def kernel_step_masks(cfg, torch_masks, p, seed, attn_site0, ffn_site0, B, S1, mem, device="cpu"):
    """Every mask of one Tiger.forward / forward_jagged step in the reference's call order.  torch_masks: the F.dropout masks in the
    order tiger.py draws them (forward: the two input dropouts, then per encoder block dropout1, per decoder block dropout1 and
    dropout_cross; forward_jagged draws the decoder input's after the encoder's); attn_site0 / ffn_site0: t5_attention._CALLS["n"] / tiger._SITES["n"] before the step (each attention call takes
    the next site, each FFN the next two); S1 the decoder length; mem = ("padded", Lm) or ("packed", T, max_len)."""
    H, D = cfg["num_heads"], cfg["attn_dim"]
    n = cfg["n_layers"] // 2
    packed = mem[0] == "packed"
    tm = list(torch_masks)
    if packed:                                          # forward_jagged runs the encoder before it draws the decoder input's mask
        tm = tm[:1] + tm[1 + n:2 + n] + tm[1:1 + n] + tm[2 + n:]
    tm = iter(tm)
    out = [next(tm), next(tm)]
    sites = {"a": attn_site0, "f": ffn_site0}

    def attn(kind, *shape):
        sites["a"] += 1
        fn = {"padded": attn_mask_padded, "self": attn_mask_packed_self, "cross": attn_mask_packed_cross}[kind]
        out.append(fn(*shape, p, seed, sites["a"], device))

    def ffn(lead):
        sites["f"] += 2
        out.extend(ffn_masks(lead, D, p, seed, sites["f"], device))

    for _ in range(n):
        if packed:
            attn("self", mem[1], H, mem[2])
        else:
            attn("padded", B, H, mem[1], mem[1])
        out.append(next(tm))
        ffn((mem[1],) if packed else (B, mem[1]))
    for _ in range(n):
        attn("padded", B, H, S1, S1)
        out.append(next(tm))
        if packed:
            attn("cross", B, H, S1, mem[2])
        else:
            attn("padded", B, H, S1, mem[1])
        out.append(next(tm))
        ffn((B, S1))
    if next(tm, None) is not None:
        raise ValueError("more torch dropout masks than the step draws")
    return out
