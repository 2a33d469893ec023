"""TEST INFRASTRUCTURE - COBRA's training step restated in plain torch (genrec/models/cobra.py:379-529 with the LightT5Encoder of
genrec/modules/encoder.py:61-103), written from the math rather than copied, for any dtype and device.  In fp64 on the GPU it is the
oracle of the GPU tests and the eager baseline of scripts/bench_cobra.py (the reference tree is not on the GPU machines).  Dropout
p = 0 only."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def _ln(x, P, name, eps=1e-5):
    return F.layer_norm(x, x.shape[-1:], P[name + ".weight"], P[name + ".bias"], eps)


def _mha(x, P, pre, H, key_pad, causal):
    """softmax(q k^T / sqrt(dh) + mask) v with in_proj / out_proj; key_pad [B, L] True = ignored key"""
    B, L, D = x.shape
    q, k, v = F.linear(x, P[pre + ".in_proj_weight"], P[pre + ".in_proj_bias"]).split(D, dim=-1)
    q, k, v = (t.view(B, L, H, D // H).transpose(1, 2) for t in (q, k, v))
    s = q @ k.transpose(-1, -2) / math.sqrt(D // H)
    ban = key_pad[:, None, None, :].expand(B, H, L, L)
    if causal:
        ban = ban | torch.ones(L, L, dtype=torch.bool, device=x.device).triu(1)
    s = s.masked_fill(ban, float("-inf"))
    p = torch.softmax(s, dim=-1).nan_to_num(0.0)                   # a row without keys attends to nothing
    a = (p @ v).transpose(1, 2).reshape(B, L, D)
    return F.linear(a, P[pre + ".out_proj.weight"], P[pre + ".out_proj.bias"])


def _ffn(x, P, pre):
    return F.linear(torch.relu(F.linear(x, P[pre + ".linear1.weight"], P[pre + ".linear1.bias"])), P[pre + ".linear2.weight"],
                    P[pre + ".linear2.bias"])


def encode(P, cfg, tokens):
    """tokens [N, L] -> unit item vectors [N, d_model]"""
    N, L = tokens.shape
    pad = tokens == 0
    x = P["encoder.embedding.weight"][tokens] + P["encoder.pos_embedding.weight"][:L].unsqueeze(0)
    H = cfg["encoder_num_heads"]
    for i in range(cfg.get("encoder_n_layers", 1)):
        pre = f"encoder.encoder.layers.{i}"
        x = _ln(x + _mha(x, P, pre + ".self_attn", H, pad, False), P, pre + ".norm1")
        x = _ln(x + _ffn(x, P, pre), P, pre + ".norm2")
    x = _ln(x, P, "encoder.layer_norm")
    keep = (~pad).unsqueeze(-1).to(x.dtype)
    pooled = (x * keep).sum(1) / keep.sum(1).clamp(min=1e-9)
    return F.normalize(F.linear(pooled, P["encoder.proj.weight"], P["encoder.proj.bias"]), dim=-1)


def forward(P, cfg, input_ids, encoder_input_ids, temperature=0.2):
    """-> dict of the CobraOutput fields"""
    C = cfg.get("n_codebooks", 3)
    V = cfg["id_vocab_size"]
    pad_id = V * C
    B, TC = input_ids.shape
    T = TC // C
    dev = input_ids.device
    vecs = encode(P, cfg, encoder_input_ids.reshape(B * T, -1)).view(B, T, -1)
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
        h = _ln(h + _mha(h, P, pre + ".self_attn", H, ~mask, True), P, pre + ".norm1")
        h = _ln(h + P[pre + ".multihead_attn.out_proj.bias"], P, pre + ".norm2")
        h = _ln(h + _ffn(h, P, pre), P, pre + ".norm3")
    loss_sparse = 0.0
    correct = torch.zeros((), dtype=torch.long, device=dev)
    total = torch.zeros((), dtype=torch.long, device=dev)
    item_ok = torch.ones(B, T - 1, dtype=torch.bool, device=dev)
    nxt = torch.arange(1, T, device=dev)
    for c in range(C):
        rows = (nxt - 1) * (C + 1) + C if c == 0 else nxt * (C + 1) + c - 1
        target = input_ids[:, nxt * C + c]
        logits = F.linear(h[:, rows], P[f"sparse_head.{c}.weight"], P[f"sparse_head.{c}.bias"])
        ok = target != pad_id
        ce = F.cross_entropy(logits.reshape(-1, V), target.reshape(-1), ignore_index=pad_id, reduction="sum")
        loss_sparse = loss_sparse + ce / ok.sum().clamp(min=1)
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
                codebook_entropy=-(prob * prob.add(1e-12).log()).sum(1).mean())


def step(params, cfg, input_ids, encoder_input_ids, dtype=torch.float64, device="cpu"):
    """forward + backward of the loss -> (outputs, grads by parameter name)"""
    P = {k: v.detach().to(device=device, dtype=dtype if v.is_floating_point() else v.dtype).requires_grad_(v.is_floating_point())
         for k, v in params.items() if k not in ("feat_queue", "queue_ptr")}
    out = forward(P, cfg, input_ids.to(device), encoder_input_ids.to(device))
    out["loss"].backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in P.items()}
    return {k: v.detach() for k, v in out.items()}, grads
