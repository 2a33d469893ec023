"""One COBRA training step at the trainer's shape (genrec/trainers/cobra_trainer.py:92-135, dropout 0.1): forward, backward and
torch's fused AdamW, timed with CUDA events, native (genrec_b200.cobra.Cobra) against the torch restatement of tests/cobra_reference.py
in eager fp32 and under bf16 autocast (dropout 0 there: the restatement has none; the native step keeps it).  Batches of B = 32 and
256 users with every user at 20 items or item counts geometric with mean 9 capped at 20, texts of 128 tokens or uniform on [16, 64].
Also times encode_items over 12,101 texts and reports peak memory.  Prints one JSON line per row.

--profile runs instead, in a separate process so that tracing does not slow the timed steps: one native step of each workload at
the largest batch under torch.profiler, with its kernel time per step split by stage (the families of kernels each stage runs)."""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tests import cobra_params as cp  # noqa: E402
from tests import cobra_reference as cr  # noqa: E402


def batch(B, items, texts, g):
    if items == "full":
        n = [20] * B
    else:
        # geometric on {1, 2, ...} with mean 9, capped at 20, from the seeded generator
        u = torch.rand(B, generator=g, dtype=torch.float64)
        n = (torch.log1p(-u) / torch.log1p(torch.tensor(-1 / 9, dtype=torch.float64))).ceil().clamp(1, 20).long().tolist()
    lens = [128] if texts == "full" else torch.randint(16, 65, (64,), generator=g).tolist()
    return cp.batch(cp.TRAINER, items=n, text_lens=lens, L=128, seed=int(torch.randint(0, 1 << 30, (1,), generator=g)))


# stage of a kernel, from its name: the first stage with a pattern whose substrings are all in the name
STAGES = (("encoder attention (T5 core, head dim 96)", (("t5_attn", "<96"),)), ("decoder attention (T5 core)", (("t5_attn",),)),
          ("T5 dK/dV partial sums", (("t5_dkdv",),)),
          ("GEMMs and their ordered sums", (("tc_gemm",), ("tn_group",), ("tn_finish",), ("colsum",), ("det_finish",))),
          ("LayerNorms", (("ln_fwd",), ("ln_bwd",))), ("text pooling", (("seg_ln_mean",),)), ("text packing", (("cobra_text",),)),
          ("InfoNCE and L2 norms", (("infonce",), ("l2norm",), ("ce_loss_sum",))), ("bf16 casts", (("cast_",),)))


def stage_of(name):
    for stage, patterns in STAGES:
        if any(all(k in name for k in pat) for pat in patterns):
            return stage
    return "torch (gathers, residuals, dropout, cross-entropy, AdamW)"


def profile(fn, warmup):
    from torch.profiler import ProfilerActivity
    from torch.profiler import profile as tprofile
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split, kernels = {}, {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            ms = e.time_range.elapsed_us() / 1000.0
            split[stage_of(e.name)] = split.get(stage_of(e.name), 0.0) + ms
            kernels[e.name[:80]] = kernels.get(e.name[:80], 0.0) + ms
    top = sorted(kernels.items(), key=lambda kv: -kv[1])[:12]
    return ({k: round(v, 2) for k, v in sorted(split.items(), key=lambda kv: -kv[1])}, [(k, round(v, 2)) for k, v in top])


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / steps, torch.cuda.max_memory_allocated() / 2**30


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--batches", default="32,256")
    args = ap.parse_args()
    from genrec_b200.cobra import Cobra
    dev = "cuda"
    cfg = dict(cp.TRAINER, decoder_dropout=0.1)
    P = cp.cobra_params(cp.shapes(cp.TRAINER), 0)
    model = Cobra(**cfg)
    model.load_state_dict(P)
    model = model.to(dev).train()
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4, weight_decay=0.01, fused=True)
    ref = {k: torch.nn.Parameter(v.to(dev)) for k, v in P.items() if k not in ("feat_queue", "queue_ptr")}
    ropt = torch.optim.AdamW(ref.values(), lr=1e-4, weight_decay=0.01, fused=True)
    info = dict(gpu=torch.cuda.get_device_name(0))
    g = torch.Generator().manual_seed(0)
    batches = [int(b) for b in args.batches.split(",")]
    for B in batches[-1:] if args.profile else batches:
        for items, texts in (("geometric", "short"), ("full", "full")):
            ids, text = (t.to(dev) for t in batch(B, items, texts, g))

            def native():
                opt.zero_grad(set_to_none=True)
                model(ids, text).loss.backward()
                opt.step()

            def eager(autocast):
                def run():
                    ropt.zero_grad(set_to_none=True)
                    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
                        out = cr.forward(ref, cp.TRAINER, ids, text)
                    out["loss"].backward()
                    ropt.step()
                return run

            row = dict(info, B=B, items=items, texts=texts, texts_encoded=int((text[:, :, 0] != 0).sum()))
            if args.profile:
                by_stage, top = profile(native, args.warmup)
                print(json.dumps(dict(row, native_kernel_ms_by_stage=by_stage, top_kernels_ms=top)), flush=True)
                continue
            for name, fn in (("native", native), ("eager_fp32", eager(False)), ("eager_bf16_autocast", eager(True))):
                try:
                    ms, mem = timed(fn, args.steps, args.warmup)
                    row[name + "_ms"], row[name + "_peak_gib"] = round(ms, 2), round(mem, 2)
                except torch.cuda.OutOfMemoryError:
                    row[name + "_ms"] = "out of memory"
                    torch.cuda.empty_cache()
            if isinstance(row.get("native_ms"), float) and isinstance(row.get("eager_bf16_autocast_ms"), float):
                row["native_over_autocast"] = round(row["native_ms"] / row["eager_bf16_autocast_ms"], 3)
            print(json.dumps(row), flush=True)
    if args.profile:
        return
    texts = torch.randint(1, cp.TRAINER["encoder_vocab_size"], (12101, 128), generator=g)
    lens = torch.randint(16, 129, (12101,), generator=g)
    texts[torch.arange(128)[None, :] >= lens[:, None]] = 0
    texts = texts.to(dev)
    model.eval()
    with torch.no_grad():
        ms, mem = timed(lambda: model.encode_items(texts), args.steps, args.warmup)
    print(json.dumps(dict(info, encode_items_texts=12101, encode_items_ms=round(ms, 2), peak_gib=round(mem, 2))), flush=True)


if __name__ == "__main__":
    main()
