"""TEST INFRASTRUCTURE - seeded COBRA parameters and ragged batches, shared by scripts/make_golden_cobra.py (which feeds them to the
reference) and the tests (which feed them to genrec_b200.cobra.Cobra), so the trainer-shape model never has to be stored."""
from __future__ import annotations

from collections import OrderedDict

import torch

SMALL = dict(encoder_hidden_dim=192, encoder_num_heads=2, encoder_vocab_size=1000, id_vocab_size=256, n_codebooks=3, d_model=128,
             max_len=128, queue_size=64, decoder_n_layers=2, decoder_num_heads=2, decoder_dropout=0.0)
# genrec/trainers/cobra_trainer.py:92-135
TRAINER = dict(encoder_n_layers=1, encoder_hidden_dim=768, encoder_num_heads=8, encoder_vocab_size=32128, id_vocab_size=256, n_codebooks=3,
               d_model=384, max_len=1024, temperature=0.2, queue_size=1024, decoder_n_layers=8, decoder_num_heads=6, decoder_dropout=0.0)
# std of the sparse heads' biases: spread wide, so that each position's top-1 and top-5 classes lead the rest by margins far above
# the bf16 error of the logits, and the integer metrics (acc_*, recall_*) can be compared exactly
HEAD_BIAS_STD = 20.0
# users of 1, 2, 7 and 20 items (the last one the target); texts of 1, 37 and 128 tokens
ITEMS = (1, 2, 7, 20)
TEXT_LENS = (1, 37, 128)


def cobra_params(shapes, seed: int) -> "OrderedDict[str, torch.Tensor]":
    """(name, shape) pairs in state_dict order -> tensors from one CPU generator.  Matrices ~ N(0, 1 / fan_in), norm weights
    1 + N(0, 0.1^2), biases N(0, 0.1^2) (the sparse heads': N(0, HEAD_BIAS_STD^2)), embeddings N(0, 1) with id_embed's padding row zero, feat_queue unit rows, queue_ptr 0."""
    g = torch.Generator().manual_seed(seed)
    out = OrderedDict()
    for name, shape in shapes:
        shape = tuple(shape)
        if name == "queue_ptr":
            out[name] = torch.zeros(shape, dtype=torch.long)
            continue
        r = torch.randn(shape, generator=g)
        if "norm" in name and name.endswith("weight"):
            t = 1.0 + 0.1 * r
        elif name.startswith("sparse_head.") and len(shape) == 1:
            t = HEAD_BIAS_STD * r
        elif len(shape) == 1:
            t = 0.1 * r
        elif "embed" in name or name == "feat_queue":
            t = r
            if name == "cobra_emb.id_embed.weight":
                t[-1] = 0.0
            if name == "feat_queue":
                t = torch.nn.functional.normalize(t, dim=-1)
        else:
            t = r / shape[-1] ** 0.5
        out[name] = t
    return out


def shapes(cfg):
    from genrec_b200.cobra import Cobra
    return [(k, tuple(v.shape)) for k, v in Cobra(**cfg).state_dict().items()]


def batch(cfg: dict, items=ITEMS, text_lens=TEXT_LENS, L: int = 128, seed: int = 0, extra_items: int = 0):
    """(input_ids [B, T*C], encoder_input_ids [B, T, L]) right-padded like cobra_collate_fn: user b has items[b] items, item t of a
    user has a text of text_lens[(b + t) % len] tokens (ids in 1 .. vocab-1), pad items have all-zero texts; T = max(items) +
    extra_items."""
    g = torch.Generator().manual_seed(seed)
    C, V = cfg["n_codebooks"], cfg["id_vocab_size"]
    B, T = len(items), max(items) + extra_items
    ids = torch.full((B, T * C), V * C, dtype=torch.long)
    text = torch.zeros(B, T, L, dtype=torch.long)
    for b, n in enumerate(items):
        ids[b, :n * C] = torch.randint(0, V, (n * C,), generator=g)
        for t in range(n):
            ln = min(text_lens[(b + t) % len(text_lens)], L)
            text[b, t, :ln] = torch.randint(1, cfg["encoder_vocab_size"], (ln,), generator=g)
    return ids, text
