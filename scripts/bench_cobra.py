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
from scripts import harness  # noqa: E402
from tests import cobra_params as cp  # noqa: E402
from tests import cobra_reference as cr  # noqa: E402


# stage of a kernel, from its name: the first stage with a key tuple whose keys are all in the name
STAGES = (("encoder attention (T5 core, head dim 96)", (("t5_attn", "<96"),)), ("decoder attention (T5 core)", (("t5_attn",),)),
          ("T5 dK/dV partial sums", (("t5_dkdv",),)),
          ("GEMMs and their ordered sums", (("tc_gemm",), ("tn_group",), ("tn_finish",), ("colsum",), ("det_finish",))),
          ("LayerNorms", (("ln_fwd",), ("ln_bwd",))), ("text pooling", (("seg_ln_mean",),)), ("text packing", (("cobra_text",),)),
          ("InfoNCE and L2 norms", (("infonce",), ("l2norm",), ("ce_loss_sum",))), ("bf16 casts", (("cast_",),)))


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
    info = harness.card(dev)
    g = torch.Generator().manual_seed(0)
    batches = [int(b) for b in args.batches.split(",")]
    for B in batches[-1:] if args.profile else batches:
        for items, texts in (("geometric", "short"), ("full", "full")):
            ids, text = (t.to(dev) for t in harness.cobra_batch(B, items, g, texts))

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
                kernels = harness.profile(native, warmup=args.warmup)
                by_stage = harness.by_stage(kernels, STAGES, "torch (gathers, residuals, dropout, cross-entropy, AdamW)")
                top = [(k, round(us / 1000.0, 2)) for k, us in list(harness.largest_first(kernels, lambda k: k[:80]).items())[:12]]
                print(json.dumps(dict(row, native_kernel_ms_by_stage=by_stage, top_kernels_ms=top)), flush=True)
                continue
            for name, fn in (("native", native), ("eager_fp32", eager(False)), ("eager_bf16_autocast", eager(True))):
                try:
                    ms, mem = harness.timed(fn, args.steps, args.warmup)
                    row[name + "_ms"], row[name + "_peak_gib"] = round(ms, 2), round(mem / 2**30, 2)
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
        ms, mem = harness.timed(lambda: model.encode_items(texts), args.steps, args.warmup)
    print(json.dumps(dict(info, encode_items_texts=12101, encode_items_ms=round(ms, 2), peak_gib=round(mem / 2**30, 2))), flush=True)


if __name__ == "__main__":
    main()
