"""COBRA generation and BeamFusion at the trainer's shape (genrec/trainers/cobra_trainer.py:92-135: d_model 384, 8 decoder layers of
6 heads, V = 256, C = 3, texts of 128 tokens), timed with CUDA events: native genrec_b200.cobra.Cobra.generate / beam_fusion against a
full-recompute torch baseline in eager fp32 and under bf16 autocast (the reference's algorithm, cobra.py:531-665: the decoder rerun
over B K copies of every history plus the tokens so far at each codebook, written batched here on tests/cobra_reference.py's layers
for users of equal length; the ragged workloads have no baseline).

Workloads: generate at B = 32 and 256 with n_beam 20 on full 20-item histories and on geometric ones (mean 9, capped at 20);
generate at n_beam 256; beam_fusion (n_candidates 10, n_beam 20) at B = 256 over N = 12,101 and 1,000,000 catalog rows.  Each row
reports the mean time per call, the peak memory, and the card's name and power limit read in the same run.

--profile runs instead, in a separate process: one native call of each workload under torch.profiler, its kernel time split by
stage."""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts import harness  # noqa: E402
from tests import cobra_generate_reference as gr  # noqa: E402
from tests import cobra_params as cp  # noqa: E402
from tests import cobra_reference as cr  # noqa: E402

STAGES = (("beam attention", (("cobra_attn",),)), ("beam selection", (("cobra_beam_topk",),)), ("catalog match", (("cobra_dense",),)),
          ("encoder attention (T5 core)", (("t5_attn", "<96"),)), ("prefill attention (T5 core)", (("t5_attn",),)),
          ("GEMMs (encoder, prefill, extension, heads)", (("tc_gemm",),)), ("LayerNorms", (("ln_fwd",),)),
          ("text pooling", (("seg_ln_mean",),)), ("L2 norms", (("l2norm",),)), ("bf16 casts", (("cast_",),)))


def baseline_generate(P, cfg, ids, text, K):
    """the reference's full-recompute beam search for users of equal length, batched over users and beams"""
    C, V = cfg["n_codebooks"], cfg["id_vocab_size"]
    B, T = text.shape[:2]
    dev = text.device
    vecs = cr.encode(P, cfg, text.reshape(B * T, -1)).view(B, T, -1)
    code = ids.view(B, T, C) + torch.arange(C, device=dev) * V
    Li = T * (C + 1)
    hist = torch.cat([P["cobra_emb.id_embed.weight"][code], vecs.unsqueeze(2)], dim=2).reshape(B, Li, -1)
    ty = (torch.arange(Li, device=dev) % (C + 1) == C).long()
    hist = hist + P["cobra_emb.pos_embed.weight"][:Li] + P["cobra_emb.type_embed.weight"][ty]
    seqs = torch.zeros(B, 1, 0, dtype=torch.long, device=dev)
    scores = torch.zeros(B, 1, dtype=hist.dtype, device=dev)
    for c in range(C):
        k = seqs.shape[1]
        x = hist.unsqueeze(1).expand(B, k, Li, -1)
        if c:
            j = torch.arange(c, device=dev)
            gen = P["cobra_emb.id_embed.weight"][seqs + j * V] + P["cobra_emb.pos_embed.weight"][Li + j] + P["cobra_emb.type_embed.weight"][0]
            x = torch.cat([x, gen], dim=2)
        out = gr._decoder(P, cfg, x.reshape(B * k, x.shape[2], -1))[:, -1]
        logp = F.log_softmax(F.linear(out, P[f"sparse_head.{c}.weight"], P[f"sparse_head.{c}.bias"]), dim=-1).view(B, k, V)
        top, flat = (scores.unsqueeze(-1) + logp).view(B, -1).topk(K, dim=-1)
        parents, tokens = flat // V, flat % V
        h_last = out.view(B, k, -1).gather(1, parents.unsqueeze(-1).expand(-1, -1, out.shape[-1]))
        seqs = torch.cat([seqs.gather(1, parents.unsqueeze(-1).expand(-1, -1, c)), tokens.unsqueeze(-1)], dim=-1)
        scores = top
    return seqs, F.normalize(h_last, dim=-1), scores


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--baseline-steps", type=int, default=2)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    from genrec_b200.cobra import Cobra
    dev = "cuda"
    cfg = dict(cp.TRAINER)
    P = cp.cobra_params(cp.shapes(cfg), 0)
    model = Cobra(**cfg)
    model.load_state_dict(P)
    model = model.to(dev).eval()
    ref = {k: v.to(dev) for k, v in P.items() if k not in ("feat_queue", "queue_ptr")}
    info = harness.card(dev)
    g = torch.Generator().manual_seed(0)
    work = [("generate", B, items, 20, None) for B in (32, 256) for items in ("full", "geometric")]
    work += [("generate", 32, "full", 256, None), ("beam_fusion", 256, "full", 20, 12101), ("beam_fusion", 256, "full", 20, 1_000_000)]
    for kind, B, items, K, N in work:
        ids, text = (t.to(dev) for t in harness.cobra_batch(B, items, g))
        row = dict(info, call=kind, B=B, items=items, n_beam=K)
        if kind == "generate":
            def native():
                model.generate(ids, text, n_candidates=K)
        else:
            vecs = torch.randn(N, cfg["d_model"], device=dev)
            sem = torch.randint(0, cfg["id_vocab_size"], (N, cfg["n_codebooks"]), device=dev)
            row["catalog"] = N

            def native():
                model.beam_fusion(ids, text, vecs, sem, n_candidates=10, n_beam=K)
        if args.profile:
            by_stage = harness.by_stage(harness.profile(native, warmup=args.warmup), STAGES,
                                        "torch (gathers, embeddings, residual adds, fusion tail)")
            print(json.dumps(dict(row, native_kernel_ms_by_stage=by_stage)), flush=True)
            continue
        ms, mem = harness.timed(native, args.steps, args.warmup)
        row["native_ms"], row["native_peak_gib"] = round(ms, 2), round(mem / 2**30, 2)
        if kind == "generate" and items == "full":
            for name, autocast in (("eager_fp32", False), ("eager_bf16_autocast", True)):
                def base():
                    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                        baseline_generate(ref, cfg, ids, text, K)
                try:
                    ms, mem = harness.timed(base, args.baseline_steps, 1)
                    row[name + "_ms"], row[name + "_peak_gib"] = round(ms, 2), round(mem / 2**30, 2)
                except torch.cuda.OutOfMemoryError:
                    row[name + "_ms"] = "out of memory"
                    torch.cuda.empty_cache()
            if isinstance(row.get("eager_bf16_autocast_ms"), float):
                row["native_over_autocast"] = round(row["native_ms"] / row["eager_bf16_autocast_ms"], 3)
        print(json.dumps(row), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
