"""COBRA serving from a paged pool at the trainer's shape (d_model 384, 8 decoder layers of 6 heads, V = 256, C = 3, texts of 128
tokens), timed with CUDA events: Cobra.extend_users + generate_users / beam_fusion_users against Cobra.generate / beam_fusion on the
same histories, the two alternated call by call in one process, medians reported.

Workloads (each row: the pool path's median, the native path's, their ratio, the pool's K | V bytes held = items (C+1) layers 2
d_model 2, and the peak memory of each path, which counts the model, the row's inputs and pool, and for fusion_1m its catalog):
  extend1      B = 256 users whose pool holds 20 full items; extend_users by 1 item, then generate_users(n_candidates=20), against
               generate on the 21-item histories
  extend1_k256 the same at B = 32 with n_beam 256
  prefill      extend_users of the full 20-item histories into an empty pool, then generate_users(20), against generate on them
  fusion_1m    beam_fusion_users (n_candidates 10, n_beam 20) over 1,000,000 catalog rows on 21-item pools, against beam_fusion
  geometric    B = 256 geometric histories (mean 9, capped at 20) in the pool, 1 new item + generate_users(20); no comparison

Between timed pool calls the users are released and their histories re-extended (untimed), so every call sees the same pool.
--profile prints, per workload, one pool call's kernel time split by stage under torch.profiler instead."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts import harness  # noqa: E402
from tests import cobra_params as cp  # noqa: E402

STAGES = (("paged attention", (("cobra_attn",),)), ("K | V scatter", (("cobra_kv_scatter",),)),
          ("beam steps (selection)", (("cobra_beam_topk",),)), ("catalog match", (("cobra_dense",),)),
          ("encoder attention (T5 core)", (("t5_attn",),)), ("GEMMs", (("tc_gemm",),)), ("LayerNorms", (("ln_fwd",),)),
          ("text pooling", (("seg_ln_mean",),)), ("L2 norms", (("l2norm",),)), ("bf16 casts", (("cast_",),)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    from genrec_b200.cobra import Cobra
    dev = "cuda"
    cfg = dict(cp.TRAINER)
    C, D, layers = cfg["n_codebooks"], cfg["d_model"], cfg["decoder_n_layers"]
    model = Cobra(**cfg)
    model.load_state_dict(cp.cobra_params(cp.shapes(cfg), 0))
    model = model.to(dev).eval()
    info = harness.card(dev)
    g = torch.Generator().manual_seed(0)
    work = [("extend1", 256, "full", 20), ("extend1_k256", 32, "full", 256), ("prefill", 256, "full", 20), ("fusion_1m", 256, "full", 20),
            ("geometric", 256, "geometric", 20)]
    for name, B, items, K in work:
        ids, text = harness.cobra_batch(B, items, g)                         # 20 items (or geometric), plus one new item below
        new_ids, new_text = cp.batch(cfg, items=[1] * B, text_lens=[128], L=128, seed=1)
        n_hist = (ids.view(B, -1, C)[:, :, C - 1] != model.pad_id).sum(1)
        # the new item right after each user's real ones, so that a geometric history stays right-padded
        full_ids = torch.full((B, 21 * C), model.pad_id, dtype=torch.long)
        full_text = torch.zeros(B, 21, 128, dtype=torch.long)
        for b, n in enumerate(n_hist.tolist()):
            full_ids[b, :n * C], full_ids[b, n * C:(n + 1) * C] = ids[b, :n * C], new_ids[b]
            full_text[b, :n], full_text[b, n] = text[b, :n], new_text[b, 0]
        ids, text, new_ids, new_text, full_ids, full_text = (t.to(dev) for t in (ids, text, new_ids, new_text, full_ids, full_text))
        users = list(range(B))
        pool = model.new_pool(max_users=B, num_pages=B * 2, page_size=64)

        def fill(with_new):
            pool.release(users)
            model.extend_users(pool, users, ids, text)
            if with_new:
                model.extend_users(pool, users, new_ids, new_text)

        if name == "prefill":
            setup, pool_call = (lambda: pool.release(users)), (lambda: (model.extend_users(pool, users, ids, text),
                                                                        model.generate_users(pool, users, n_candidates=K)))
            native = lambda: model.generate(ids, text, n_candidates=K)                 # noqa: E731
            held = int(n_hist.sum()) * (C + 1) * layers * 2 * D * 2
        elif name == "fusion_1m":                                    # the 1.5 GB catalog lives only for this row's peaks
            vecs = torch.randn(1_000_000, D, device=dev)
            sem = torch.randint(0, cfg["id_vocab_size"], (1_000_000, C), device=dev)
            setup, pool_call = (lambda: fill(True)), (lambda: model.beam_fusion_users(pool, users, vecs, sem, n_candidates=10, n_beam=K))
            native = lambda: model.beam_fusion(full_ids, full_text, vecs, sem, n_candidates=10, n_beam=K)   # noqa: E731
            held = int(n_hist.sum() + B) * (C + 1) * layers * 2 * D * 2
        else:
            setup, pool_call = (lambda: fill(False)), (lambda: (model.extend_users(pool, users, new_ids, new_text),
                                                                model.generate_users(pool, users, n_candidates=K)))
            native = (lambda: model.generate(full_ids, full_text, n_candidates=K)) if name != "geometric" else None
            held = int(n_hist.sum() + B) * (C + 1) * layers * 2 * D * 2
        row = dict(info, workload=name, B=B, items=items, n_beam=K, pool_kv_bytes=held)
        if args.profile:
            setup()
            pool_call()
            setup()
            kernels = harness.profile(pool_call, warmup=0)
            by_stage = harness.by_stage(kernels, STAGES, "torch (gathers, embeddings, residual adds, fusion tail)")
            print(json.dumps(dict(row, pool_kernel_ms_by_stage=by_stage)), flush=True)
            continue
        tp, tn = [], []
        for i in range(args.warmup + args.steps):
            setup()
            a = harness.timed(pool_call, 1, 0)[0]
            b = harness.timed(native, 1, 0)[0] if native else None
            if i >= args.warmup:
                tp.append(a)
                if native:
                    tn.append(b)
        setup()
        row["pool_ms"] = round(statistics.median(tp), 2)
        base = torch.cuda.memory_allocated() / 2**30
        row["pool_peak_gib"] = round(harness.peak(pool_call) / 2**30, 2)
        row["pool_held_gib_after"] = round(base, 2)
        if native:
            row["native_ms"] = round(statistics.median(tn), 2)
            row["native_peak_gib"] = round(harness.peak(native) / 2**30, 2)
            row["pool_over_native"] = round(row["pool_ms"] / row["native_ms"], 3)
        print(json.dumps(row), flush=True)
        del pool
        vecs = sem = None
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
