"""TEST INFRASTRUCTURE - seeded TIGER parameters, shared by scripts/make_golden_tiger.py (which feeds them to the reference) and the
tests (which feed them to genrec_b200.tiger.Tiger), so the published-shape model (13 M parameters) never has to be stored; and the
GPU tests' seeded models and their padded and packed batches."""
from __future__ import annotations

from collections import OrderedDict

import numpy as np
import torch

DEV = torch.device("cuda:0")

SMALL = dict(embedding_dim=64, attn_dim=64, dropout=0.0, num_heads=2, n_layers=2, num_item_embeddings=16, num_user_embeddings=50,
             sem_id_dim=3)
# config/tiger/amazon/tiger.gin
PUBLISHED = dict(embedding_dim=128, attn_dim=384, dropout=0.0, num_heads=6, n_layers=8, num_item_embeddings=256, num_user_embeddings=10000,
                 sem_id_dim=3)


def tiger_params(shapes, seed: int, padding_key: str = "sem_id_embedding.emb.weight") -> "OrderedDict[str, torch.Tensor]":
    """shapes: (name, shape) pairs in state_dict order -> fp32 tensors from one CPU generator.  Matrices ~ N(0, 1 / fan_in), norm
    weights 1 + N(0, 0.1^2), relative-bias tables N(0, 0.5^2), embeddings N(0, 1) with the padding row (the last) zero."""
    g = torch.Generator().manual_seed(seed)
    out = OrderedDict()
    for name, shape in shapes:
        shape = tuple(shape)
        r = torch.randn(shape, generator=g)
        if "rel_bias" in name:
            t = 0.5 * r
        elif len(shape) == 1 and name != "bos_embedding":
            t = 1.0 + 0.1 * r
        elif "emb" in name or name == "bos_embedding":
            t = r
            if name == padding_key:
                t[-1] = 0.0
        else:
            t = r / shape[-1] ** 0.5
        out[name] = t
    return out


def batch(cfg: dict, B: int, n_items: int, seed: int):
    """A padded batch: item histories of n_items items (n_items * sem_id_dim tokens), right-padded with the padding id; the first
    user has the full history, later users progressively shorter ones.  Returns a dict of CPU int64 tensors."""
    g = torch.Generator().manual_seed(seed)
    C, E = cfg["sem_id_dim"], cfg["num_item_embeddings"]
    N = n_items * C
    users = torch.randint(0, 10 * cfg["num_user_embeddings"], (B, 1), generator=g)
    items = torch.randint(0, E, (B, N), generator=g)
    types = torch.arange(N).remainder(C).unsqueeze(0).expand(B, -1).contiguous()
    mask = torch.ones(B, N, dtype=torch.long)
    for b in range(1, B):
        keep = max(1, n_items - (b * n_items) // B) * C
        mask[b, keep:] = 0
    items[mask == 0] = C * E                       # the padding id, with token type 0 (tiger.py:471-476)
    types = torch.where(mask == 0, torch.zeros_like(types), types)
    target = torch.randint(0, E, (B, C), generator=g)
    target_types = torch.arange(C).unsqueeze(0).expand(B, -1).contiguous()
    return dict(user_input_ids=users, item_input_ids=items, token_type_ids=types, target_input_ids=target,
                target_token_type_ids=target_types, seq_mask=mask)


# ------------------------------------------------------------------------------------------------ models and batches on the GPU
def _model(cfg, seed=7):
    from genrec_b200.tiger import Tiger
    m = Tiger(**cfg)
    m.load_state_dict(tiger_params([(k, v.shape) for k, v in m.state_dict().items()], seed))
    return m.to(DEV)


def _padded_and_packed(cfg, B, n_items, seed, lengths=None, num_tokens=None):
    """batch's padded batch (or one with the given item counts) and the same users packed by data.pack_tiger (into num_tokens
    rows, the rest idle, when given)"""
    from genrec_b200.data import pack_tiger
    b = batch(cfg, B, n_items, seed)
    C, E = cfg["sem_id_dim"], cfg["num_item_embeddings"]
    if lengths is not None:                        # redraw the histories at these item counts (pads: the padding id, type 0)
        N = n_items * C
        mask = (torch.arange(N)[None, :] < torch.tensor(lengths)[:, None] * C).long()
        ids = torch.randint(0, E, (B, N), generator=torch.Generator().manual_seed(seed + 1))
        types = torch.arange(N).remainder(C).unsqueeze(0).expand(B, -1)
        b["seq_mask"] = mask
        b["item_input_ids"] = torch.where(mask == 0, torch.full_like(ids, C * E), ids)
        b["token_type_ids"] = torch.where(mask == 0, torch.zeros_like(ids), types)
    lens = b["seq_mask"].sum(1)
    toks = torch.cat([b["item_input_ids"][i, :int(lens[i])] for i in range(B)])
    off = torch.zeros(B + 1, dtype=torch.int64)
    off[1:] = lens.cumsum(0)
    pk = pack_tiger(b["user_input_ids"].view(-1).to(DEV), toks.to(DEV), off.to(DEV), b["target_input_ids"].to(DEV), max_items=n_items,
                    num_tokens=num_tokens)
    # the padded batch at the width of its longest history, as pad_collate makes it
    width = int(lens.max())
    padded = {k: v.to(DEV) for k, v in b.items()}
    for k in ("item_input_ids", "token_type_ids", "seq_mask"):
        padded[k] = padded[k][:, :width].contiguous()
    return padded, pk


def _geometric_lengths(B, seed, cap=20, mean=9.0):
    g = np.random.default_rng(seed)
    return np.minimum(g.geometric(1.0 / mean, B), cap).tolist()
