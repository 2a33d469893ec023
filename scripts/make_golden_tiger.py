"""Generate tests/golden/tiger_*.pt from the UNMODIFIED reference Tiger (needs the reference tree, see oracle/ref_loader.py).

    python scripts/make_golden_tiger.py

Parameters come from tests/tiger_params.py (seeded, rebuilt by the tests), so no fixture stores a state_dict; each stores the
reference's parameter names and shapes instead.  Every file stays under 1 MB (tests/conftest.py merges <stem>.<key>.pt parts).
  tiger_small.pt       attn_dim 64, 2 heads, 2 layers: forward (logits, loss, every parameter gradient), _encode_context and
                       _decode_step on a padded batch
  tiger_published.pt   config/tiger/amazon/tiger.gin shape, B = 4, 20-item padded histories: logits, loss, the gradients of the
                       vectors in full and of every matrix at 1,024 seeded positions (with its Frobenius norm)
  tiger_generate.pt    generate at the published shape, K = 10, a trie of 2,000 items, with the torch.multinomial draws recorded; the
                       seed is the first whose top K + 1 distinct candidate sequences differ in score by at least MARGIN at every step
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from oracle import tiger_decode as od  # noqa: E402
from tests import tiger_params as tp  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
SAMPLES = 1024
MARGIN = 1e-3


def _model(tg, cfg, seed):
    m = tg.Tiger(**cfg)
    shapes = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    m.load_state_dict(tp.tiger_params(shapes, seed), strict=True)
    return m, shapes


def _fwd(m, b):
    m.zero_grad()
    out = m(**b)
    out.loss.backward()
    return out


def positions(numel: int, seed: int) -> torch.Tensor:
    return torch.randperm(numel, generator=torch.Generator().manual_seed(seed))[:SAMPLES].sort().values


def golden_small(tg):
    cfg, pseed, bseed = tp.SMALL, 1, 2
    m, shapes = _model(tg, cfg, pseed)
    b = tp.batch(cfg, 4, 5, bseed)
    out = _fwd(m, b)
    grads = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
    with torch.no_grad():
        memory, mpad = m._encode_context(b["user_input_ids"], b["item_input_ids"], b["token_type_ids"], b["seq_mask"])
        types = torch.arange(2).unsqueeze(0).expand(4, -1)
        step = m._decode_step(memory, mpad, b["target_input_ids"][:, :2], types)
        step0 = m._decode_step(memory, mpad, None, None)
    big = {n for n, g in grads.items() if g.numel() >= 65536}
    torch.save(dict(cfg=cfg, param_seed=pseed, batch_seed=bseed, B=4, n_items=5, shapes=shapes, logits=out.logits.detach().clone(),
                    loss=out.loss.detach().clone(), grads={n: g for n, g in grads.items() if n not in big}, memory=memory.clone(),
                    memory_mask=mpad.clone(), step_logits=step.clone(), step0_logits=step0.clone()), os.path.join(OUT, "tiger_small.pt"))
    for n in sorted(big):            # the FFN matrices, one part each
        torch.save({n: grads[n]}, os.path.join(OUT, "tiger_small.grads_" + n.replace(".", "_") + ".pt"))


def golden_published(tg):
    cfg, pseed, bseed = tp.PUBLISHED, 3, 4
    m, shapes = _model(tg, cfg, pseed)
    b = tp.batch(cfg, 4, 20, bseed)
    out = _fwd(m, b)
    vec, sampled = {}, {}
    for i, (n, p) in enumerate(m.named_parameters()):
        if p.grad is None:
            continue
        if p.grad.dim() == 1 or p.grad.shape[-1] == 1:
            vec[n] = p.grad.clone()
        else:
            pos = positions(p.grad.numel(), 100 + i)
            sampled[n] = dict(pos=pos, values=p.grad.reshape(-1)[pos].clone(), frob=p.grad.norm().item())
    torch.save(dict(cfg=cfg, param_seed=pseed, batch_seed=bseed, B=4, n_items=20, shapes=shapes, logits=out.logits.detach().clone(),
                    loss=out.loss.detach().clone(), vec_grads=vec, sampled_grads=sampled), os.path.join(OUT, "tiger_published.pt"))


def _margin(step_logits, draws, B, K, num_emb, temperature, valid):
    """Smallest gap between adjacent scores among each user's top K + 1 candidates, over all steps (the reference's beam order is
    decided there), replayed with the oracle restatement of the decode loop."""
    root = od.build_trie(valid)
    beam_seqs = torch.empty(B, K, 0, dtype=torch.long)
    beam_logps = torch.zeros(B, K)
    nodes = [[root] * K for _ in range(B)]
    KK = draws[0].shape[1]
    gap = float("inf")
    for step, (logits, cand) in enumerate(zip(step_logits, draws)):
        off = step * num_emb
        _, logp = od.masked_log_softmax(logits, nodes, B, K, off, num_emb, temperature, True)
        cand_logp = torch.gather(logp, 1, cand).view(B, K, KK)
        total = (beam_logps.unsqueeze(-1) + cand_logp).view(B, -1)
        tok = (cand - off).view(B, -1)
        for b in range(B):
            scores, order = total[b].sort(descending=True, stable=True)
            seen, top = set(), []
            for s, j in zip(scores.tolist(), order.tolist()):
                key = tuple(beam_seqs[b, j // KK].tolist()) + (tok[b, j].item(),)
                if key not in seen:            # identical sequences (all beams at step 0) are one candidate
                    seen.add(key)
                    top.append(s)
                if len(top) == K + 1:
                    break
            gap = min([gap] + [x - y for x, y in zip(top[:-1], top[1:])])
        beam_seqs, beam_logps, nodes = od.select(beam_seqs, beam_logps, (cand - off).view(B, K, KK), cand_logp, nodes, root)
    return gap


def golden_generate(tg, B=3, K=10, temperature=0.2):
    cfg, pseed = tp.PUBLISHED, 3
    m, _ = _model(tg, cfg, pseed)
    m.eval()
    valid = torch.randint(0, cfg["num_item_embeddings"], (2000, cfg["sem_id_dim"]), generator=torch.Generator().manual_seed(7))
    for seed in range(10, 400):
        b = tp.batch(cfg, B, 20, seed)
        step_logits, draws = [], []
        orig_step, orig_multi = m._decode_step, torch.multinomial

        def rec_step(*a, **k):
            out = orig_step(*a, **k)
            step_logits.append(out.detach().clone())
            return out

        def rec_multi(*a, **k):
            out = orig_multi(*a, **k)
            draws.append(out.clone())
            return out

        m._decode_step, torch.multinomial = rec_step, rec_multi
        m.trie_root = None
        torch.manual_seed(seed)
        try:
            with torch.no_grad():
                out = m.generate(b["user_input_ids"], b["item_input_ids"], b["token_type_ids"], b["seq_mask"], temperature=temperature,
                                 n_top_k_candidates=K, valid_item_ids=valid)
        finally:
            torch.multinomial = orig_multi
            del m._decode_step
        gap = _margin(step_logits, draws, B, K, cfg["num_item_embeddings"], temperature, valid)
        print("generate seed", seed, "margin", gap)
        if gap >= MARGIN:
            torch.save(dict(cfg=cfg, param_seed=pseed, batch_seed=seed, B=B, K=K, n_items=20, temperature=temperature, valid_item_ids=valid,
                            draws=draws, sem_ids=out.sem_ids.clone(), log_probas=out.log_probas.clone(), margin=gap),
                       os.path.join(OUT, "tiger_generate.pt"))
            return
    raise RuntimeError("no seed with the required margin")


def main():
    assert ref_loader.available(), "reference tree not found"
    tg = ref_loader.ref_tiger()
    golden_small(tg)
    golden_published(tg)
    golden_generate(tg)
    for f in sorted(os.listdir(OUT)):
        if f.startswith("tiger_") and not f.startswith("tiger_decode"):
            print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()
