"""TEST INFRASTRUCTURE - COBRA's training step restated in plain torch (genrec/models/cobra.py:379-529 with the LightT5Encoder of
genrec/modules/encoder.py:61-103), written from the math rather than copied, for any dtype and device.  In fp64 on the GPU it is the
oracle of the GPU tests and the eager baseline of scripts/bench_cobra.py (the reference tree is not on the GPU machines).

Dropout: with `masks` (a list of keep-scale tensors: 0 where dropped, the keep scale elsewhere) every dropout of the reference is
applied in its call order, on the reference's padded shapes.  Per encoder layer (nn.TransformerEncoderLayer, post-LN): the attention
probabilities [N, H, L, L], dropout1 [N, L, D], the FFN's hidden dropout [N, L, F], dropout2 [N, L, D].  Per decoder layer: the
self-attention probabilities [B, H, Li, Li], dropout1, dropout2 on the cross-attention output (the out_proj bias: the memory is
empty, so its attention has no probabilities to drop), the hidden dropout, dropout3.  masks=None is dropout 0.  `kernel_step_masks`
rebuilds that list for one step of genrec_b200.cobra.Cobra from its two dropout seeds and the masks its torch-side dropouts drew."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

MARGIN = 5e-2               # logit units: a top-1 lead below this may flip under bf16 rounding


def _ln(x, P, name, eps=1e-5):
    return F.layer_norm(x, x.shape[-1:], P[name + ".weight"], P[name + ".bias"], eps)


def _keep(masks, shape):
    if masks is None:
        return None
    k = next(masks, None)
    if k is None:
        raise ValueError("fewer masks than the step's dropouts")
    if tuple(k.shape) != tuple(shape):
        raise ValueError(f"mask {tuple(k.shape)} for a dropout of {tuple(shape)}")
    return k


def _drop(x, masks):
    k = _keep(masks, x.shape)
    return x if k is None else x * k.to(x.dtype)


def _mha(x, P, pre, H, key_pad, causal, masks=None):
    """softmax(q k^T / sqrt(dh) + mask) v with in_proj / out_proj; key_pad [B, L] True = ignored key"""
    B, L, D = x.shape
    q, k, v = F.linear(x, P[pre + ".in_proj_weight"], P[pre + ".in_proj_bias"]).split(D, dim=-1)
    q, k, v = (t.view(B, L, H, D // H).transpose(1, 2) for t in (q, k, v))
    s = q @ k.transpose(-1, -2) / math.sqrt(D // H)
    ban = key_pad[:, None, None, :].expand(B, H, L, L)
    if causal:
        ban = ban | torch.ones(L, L, dtype=torch.bool, device=x.device).triu(1)
    s = s.masked_fill(ban, float("-inf"))
    p = _drop(torch.softmax(s, dim=-1).nan_to_num(0.0), masks)    # a row without keys attends to nothing
    a = (p @ v).transpose(1, 2).reshape(B, L, D)
    return F.linear(a, P[pre + ".out_proj.weight"], P[pre + ".out_proj.bias"])


def _ffn(x, P, pre, masks=None):
    h = _drop(torch.relu(F.linear(x, P[pre + ".linear1.weight"], P[pre + ".linear1.bias"])), masks)
    return _drop(F.linear(h, P[pre + ".linear2.weight"], P[pre + ".linear2.bias"]), masks)


def encode(P, cfg, tokens, masks=None):
    """tokens [N, L] -> unit item vectors [N, d_model]; masks: an iterator over the encoder's keep-scale tensors, or None"""
    N, L = tokens.shape
    pad = tokens == 0
    x = P["encoder.embedding.weight"][tokens] + P["encoder.pos_embedding.weight"][:L].unsqueeze(0)
    H = cfg["encoder_num_heads"]
    for i in range(cfg.get("encoder_n_layers", 1)):
        pre = f"encoder.encoder.layers.{i}"
        x = _ln(x + _drop(_mha(x, P, pre + ".self_attn", H, pad, False, masks), masks), P, pre + ".norm1")
        x = _ln(x + _ffn(x, P, pre, masks), P, pre + ".norm2")
    x = _ln(x, P, "encoder.layer_norm")
    keep = (~pad).unsqueeze(-1).to(x.dtype)
    pooled = (x * keep).sum(1) / keep.sum(1).clamp(min=1e-9)
    return F.normalize(F.linear(pooled, P["encoder.proj.weight"], P["encoder.proj.bias"]), dim=-1)


def forward(P, cfg, input_ids, encoder_input_ids, temperature=0.2, masks=None):
    """-> dict of the CobraOutput fields, and "near": the counted positions whose top-1 logit leads the next by less than MARGIN
    (where a bf16 model's argmax may differ)"""
    masks = iter(masks) if masks is not None else None
    C = cfg.get("n_codebooks", 3)
    V = cfg["id_vocab_size"]
    pad_id = V * C
    B, TC = input_ids.shape
    T = TC // C
    dev = input_ids.device
    vecs = encode(P, cfg, encoder_input_ids.reshape(B * T, -1), masks).view(B, T, -1)
    sparse_mask = (input_ids != pad_id).view(B, T, C)
    mask = torch.cat([sparse_mask, sparse_mask[:, :, -1:]], dim=2).reshape(B, -1)
    code = input_ids.view(B, T, C) + torch.arange(C, device=dev) * V
    tok = P["cobra_emb.id_embed.weight"][torch.where(sparse_mask, code, torch.full_like(code, pad_id))]
    h = torch.cat([tok, vecs.unsqueeze(2)], dim=2).reshape(B, T * (C + 1), -1)
    Li = T * (C + 1)
    ty = (torch.arange(Li, device=dev) % (C + 1) == C).long()
    m = mask.unsqueeze(-1).to(h.dtype)
    h = (h + P["cobra_emb.pos_embed.weight"][:Li] + P["cobra_emb.type_embed.weight"][ty]) * m
    H = cfg["decoder_num_heads"]
    for i in range(cfg["decoder_n_layers"]):
        pre = f"decoder.decoder.layers.{i}"
        h = _ln(h + _drop(_mha(h, P, pre + ".self_attn", H, ~mask, True, masks), masks), P, pre + ".norm1")
        h = _ln(h + _drop(P[pre + ".multihead_attn.out_proj.bias"].expand_as(h), masks), P, pre + ".norm2")
        h = _ln(h + _ffn(h, P, pre, masks), P, pre + ".norm3")
    if masks is not None:
        if next(masks, None) is not None:
            raise ValueError("more masks than the step's dropouts")
    loss_sparse = 0.0
    correct = torch.zeros((), dtype=torch.long, device=dev)
    total = torch.zeros((), dtype=torch.long, device=dev)
    near = torch.zeros((), dtype=torch.long, device=dev)
    item_ok = torch.ones(B, T - 1, dtype=torch.bool, device=dev)
    nxt = torch.arange(1, T, device=dev)
    for c in range(C):
        rows = (nxt - 1) * (C + 1) + C if c == 0 else nxt * (C + 1) + c - 1
        target = input_ids[:, nxt * C + c]
        logits = F.linear(h[:, rows], P[f"sparse_head.{c}.weight"], P[f"sparse_head.{c}.bias"])
        ok = target != pad_id
        ce = F.cross_entropy(logits.reshape(-1, V), target.reshape(-1), ignore_index=pad_id, reduction="sum")
        loss_sparse = loss_sparse + ce / ok.sum().clamp(min=1)
        top2 = logits.detach().topk(2, -1).values
        near = near + ((top2[..., 0] - top2[..., 1] < MARGIN) & ok).sum()
        top1 = logits.argmax(-1) == target
        correct = correct + (top1 & ok).sum()
        total = total + ok.sum()
        item_ok &= top1 | ~ok
        if c == 0:
            valid0 = ok
    loss_sparse = loss_sparse / C
    valid = mask[:, C + 1::C + 1]
    pred = F.normalize(h[:, nxt * (C + 1) + C - 1][valid], dim=-1)
    gt = F.normalize(vecs[:, 1:].detach()[valid], dim=-1)
    user = torch.arange(B, device=dev).unsqueeze(1).expand(B, T - 1)[valid]
    same = (user[:, None] == user[None, :]) & ~torch.eye(user.numel(), dtype=torch.bool, device=dev)
    sim = (pred @ gt.T / temperature).masked_fill(same, float("-inf"))
    loss_dense = F.cross_entropy(sim, torch.arange(sim.shape[0], device=dev)) if sim.shape[0] else torch.full((), float("nan"), device=dev)
    usage = torch.stack([F.one_hot(input_ids[:, c::3], pad_id + 1).sum((0, 1)).to(h.dtype) for c in range(C)])
    prob = usage / usage.sum(1, keepdim=True)
    return dict(loss=loss_sparse + loss_dense, loss_sparse=loss_sparse, loss_dense=loss_dense, acc_correct=correct, acc_total=total,
                recall_correct=(item_ok & valid0).sum(), recall_total=valid0.sum(),
                vec_cos_sim=F.cosine_similarity(pred, gt).mean().detach() if pred.shape[0] else torch.full((), float("nan"), device=dev),
                codebook_entropy=-(prob * prob.add(1e-12).log()).sum(1).mean(), near=near)


def step(params, cfg, input_ids, encoder_input_ids, dtype=torch.float64, device="cpu", masks=None, autocast=False):
    """forward + backward of the loss -> (outputs, grads by parameter name); autocast: under bf16 torch.autocast"""
    P = {k: v.detach().to(device=device, dtype=dtype if v.is_floating_point() else v.dtype).requires_grad_(v.is_floating_point())
         for k, v in params.items() if k not in ("feat_queue", "queue_ptr")}
    if masks is not None:
        masks = [k.to(device=device, dtype=dtype) for k in masks]
    with torch.autocast(torch.device(device).type, dtype=torch.bfloat16, enabled=autocast):
        out = forward(P, cfg, input_ids.to(device), encoder_input_ids.to(device), masks=masks)
    out["loss"].backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in P.items()}
    return {k: v.detach() for k, v in out.items()}, grads


# ------------------------------------------------------------------------------------------------ masks
def fixture_masks(shapes, mask_seed, p):
    """the keep-scale masks of a dropout fixture (scripts/make_golden_cobra_dropout.py), in call order: keep = rand >= p from one
    CPU generator seeded with mask_seed, at the kernels' keep scale"""
    from tests.attention_reference import keep_scale
    g = torch.Generator().manual_seed(mask_seed)
    return [(torch.rand(s, generator=g, dtype=torch.float64) >= p).double() * keep_scale(p)[1] for s in shapes]


def text_rows(encoder_input_ids, input_ids, pad_id, C):
    """the packed rows genrec_b200.cobra encodes: (text index, position) of every row, in row order, and the offsets [N + 1].  A text
    is its leading non-zero tokens; pad items' texts have none."""
    B, T, L = encoder_input_ids.shape
    tok = encoder_input_ids.reshape(B * T, L).cpu()
    nz = (tok != 0).long()
    lens = nz.cumprod(1).sum(1)
    lens = lens * (input_ids.view(B, T, C)[:, :, C - 1] != pad_id).reshape(-1).cpu().long()
    text = torch.arange(B * T).repeat_interleave(lens)
    offsets = torch.cat([torch.zeros(1, dtype=torch.long), lens.cumsum(0)])
    pos = torch.arange(int(offsets[-1])) - offsets[:-1].repeat_interleave(lens)
    return text, pos, offsets


def _scatter(packed, text, pos, N, L):
    """[rows, C] packed-row keep-scale values -> [N, L, C], 1 where no row is"""
    full = torch.ones(N, L, packed.shape[-1], dtype=torch.float64, device=packed.device)
    full[text.to(packed.device), pos.to(packed.device)] = packed.double()
    return full


def kernel_step_masks(params, cfg, input_ids, encoder_input_ids, p, seeds, torch_masks, device="cpu"):
    """The masks of one training step of genrec_b200.cobra.Cobra at dropout p everywhere, in the order `forward` applies them.
    seeds: the step's two dropout seeds (Cobra._seed: the encoder's, then the decoder's).  torch_masks: the keep-scale tensors its
    torch-side dropouts drew, in call order (per encoder layer dropout1 [rows, D]; per decoder layer dropout1 and dropout2
    [B, Li, D]).  The kernels' masks are restated from (seed, site):
      encoder attention   packed self-attention, row key (row H + h), site 16 i + 1, mapped into each text's [H, L, L]
      encoder FFN         hidden at site 16 i + 2, output at 16 i + 3, keyed by packed row
      decoder attention   padded causal, row key (b H + h) Li + t, site 16 i + 1
      decoder FFN         hidden at 16 i + 2, output at 16 i + 3, keyed by b Li + t"""
    from tests import dense_reference as dr
    from tests.attention_reference import attn_keep
    from tests.tiger_reference import attn_mask_packed_self
    C = cfg.get("n_codebooks", 3)
    pad_id = cfg["id_vocab_size"] * C
    B, T, L = encoder_input_ids.shape
    N = B * T
    text, pos, offsets = text_rows(encoder_input_ids, input_ids, pad_id, C)
    rows = int(offsets[-1])
    lens = (offsets[1:] - offsets[:-1]).tolist()
    mx = max(lens)
    tm = iter(torch_masks)
    out = []
    He, Hd = cfg["encoder_num_heads"], cfg["decoder_num_heads"]
    for i in range(cfg.get("encoder_n_layers", 1)):
        pre = f"encoder.encoder.layers.{i}"
        Fd, De = params[pre + ".linear1.weight"].shape
        km = attn_mask_packed_self(rows, He, mx, p, seeds[0], 16 * i + 1, device)
        att = torch.ones(N, He, L, L, dtype=torch.float64, device=device)
        for n in range(N):
            r0, ln = int(offsets[n]), lens[n]
            if ln:
                att[n, :, :ln, :ln] = km[r0:r0 + ln, :, :ln].transpose(0, 1)
        out.append(att)
        out.append(_scatter(next(tm).to(device), text, pos, N, L))
        out.append(_scatter(dr.keep(range(rows), Fd, p, seeds[0], 16 * i + 2, device), text, pos, N, L))
        out.append(_scatter(dr.keep(range(rows), De, p, seeds[0], 16 * i + 3, device), text, pos, N, L))
    Li = T * (C + 1)
    for i in range(cfg["decoder_n_layers"]):
        pre = f"decoder.decoder.layers.{i}"
        Fd, D = params[pre + ".linear1.weight"].shape
        out.append(attn_keep(B, Hd, Li, Li, p, seeds[1], 16 * i + 1, device))
        out.append(next(tm).to(device).double())
        out.append(next(tm).to(device).double())
        out.append(dr.keep(range(B * Li), Fd, p, seeds[1], 16 * i + 2, device).view(B, Li, Fd))
        out.append(dr.keep(range(B * Li), D, p, seeds[1], 16 * i + 3, device).view(B, Li, D))
    if next(tm, None) is not None:
        raise ValueError("more torch dropout masks than the step draws")
    return out
