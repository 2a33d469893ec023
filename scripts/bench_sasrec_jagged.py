"""Training step and evaluation of SASRec on a packed (jagged) batch against the left-padded batch of the same users.

Reference geometry (config/sasrec/amazon.gin): V = 12,101 items, d = 64, H = 2, 2 blocks, FFN 256, max_seq_len 50.  For each workload
one seeded batch of users is drawn as a jagged batch on the device; the padded step trains on collate_jagged of it and the packed
step on pack_jagged of it.  A step is forward, backward and the FlatAdam update, captured in a CUDA graph and replayed; the two graphs
are timed with CUDA events, alternated three times in one process (medians).  Dropout is 0, so both steps optimise the same objective:
the padded batch's targets at pad inputs (sasrec_collate_fn's shift makes the last pad row predict the first item) are zeroed, and the
first-step losses must agree to rounding.  evaluate_batch against evaluate_batch_jagged is timed the same way at B = 256, and
``--profile`` adds a torch.profiler per-kernel breakdown of one eager step of each path.

    python scripts/bench_sasrec_jagged.py [--steps 30] [--workloads geo1024,geo128,full128] [--profile geo1024]

Prints one JSON line per workload."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from scripts import harness  # noqa: E402

CFG = dict(num_items=12101, max_seq_len=50, embed_dim=64, num_heads=2, num_blocks=2, ffn_dim=256)
WORKLOADS = {   # name: (B, lengths, description, aim on packed / padded)
    "geo1024": (1024, "geometric", "lengths geometric, mean 9, capped at 50", "<= 0.5"),
    "geo128": (128, "geometric", "lengths geometric, mean 9, capped at 50", "none"),
    "full128": (128, "full", "every length 50", "within 3%"),
}
EVAL_B = 256


def jagged_batch(kind, B, V, seed, dev):
    g = torch.Generator().manual_seed(seed)
    lens = torch.full((B,), 50) if kind == "full" else harness.geometric_lengths(B, 9, 1, 50, g)
    w = torch.arange(1, V + 1, dtype=torch.float64).pow(-1.1)
    items = torch.multinomial(w, int(lens.sum()), replacement=True, generator=g) + 1
    tgt = torch.multinomial(w, B, replacement=True, generator=g) + 1
    off = torch.zeros(B + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(lens, 0)
    return items.to(dev), off.to(dev), tgt.to(dev)


def make(dev):
    from genrec_b200.optim import FlatAdam
    from genrec_b200.sasrec import SASRec
    torch.manual_seed(0)
    m = SASRec(dropout=0.0, **CFG).to(dev).train()
    return m, FlatAdam(m, lr=1e-3, betas=(0.9, 0.98))


def batches(kind, B, dev):
    from genrec_b200.data import collate_jagged, pack_jagged
    items, off, tgt = jagged_batch(kind, B, CFG["num_items"], 1234, dev)
    pad = collate_jagged(items, off, tgt, CFG["max_seq_len"])
    pad_tg = torch.where(pad["input_ids"] == 0, 0, pad["targets"])
    pk = pack_jagged(items, off, tgt, CFG["max_seq_len"])
    return pad, pad_tg, pk, tgt


def run(name, steps, dev, info, profile):
    B, kind, desc, aim = WORKLOADS[name]
    pad, pad_tg, pk, _ = batches(kind, B, dev)
    T, L = pk["input_ids"].numel(), pad["input_ids"].shape[1]
    res = {}
    for path in ("padded", "packed"):
        m, opt = make(dev)

        def step(m=m, opt=opt, path=path):
            if path == "padded":
                _, loss = m(pad["input_ids"], pad_tg)
            else:
                _, loss = m.forward_jagged(pk["input_ids"], pk["offsets"], pk["max_len"], pk["targets"])
            loss.backward()
            opt.step()
            return loss

        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()           # step_peak_mem_mb: the step's working memory above what is already resident
        torch.cuda.reset_peak_memory_stats()
        loss0 = step().item()                          # the first step's loss, from the same initial parameters on both paths
        g, _ = harness.graphed(step, 3)
        g.replay()
        torch.cuda.synchronize()
        res[path] = dict(step=step, graph=g, loss0=loss0, peak_mb=(torch.cuda.max_memory_allocated() - base) / 2 ** 20)
    times = {"padded": [], "packed": []}
    for _ in range(3):
        for path in ("padded", "packed"):
            times[path].append(harness.timed(res[path]["graph"].replay, steps, 1)[0])
    out = dict(workload=name, desc=desc, B=B, aim=aim, padded_L=L, padded_tokens=B * L, packed_tokens=T,
               padding_share=round(1 - T / (B * L), 4), **info)
    for path in ("padded", "packed"):
        ms = statistics.median(times[path])
        out[path] = dict(step_ms=round(ms, 4), runs_ms=[round(t, 4) for t in times[path]], seq_per_s=round(B / ms * 1e3, 1),
                         step_peak_mem_mb=round(res[path]["peak_mb"], 1), loss_step1=res[path]["loss0"])
    out["packed_over_padded"] = round(out["packed"]["step_ms"] / out["padded"]["step_ms"], 4)
    out["loss_rel_diff"] = abs(res["packed"]["loss0"] - res["padded"]["loss0"]) / abs(res["padded"]["loss0"])
    if profile:
        for path in ("padded", "packed"):
            res[path]["graph"].reset()
            kernels = harness.largest_first(harness.profile(res[path]["step"]), lambda k: harness.short_name(k)[:60])
            out[path]["kernels_us"] = {k: round(us, 1) for k, us in kernels.items()}
    print(json.dumps(out), flush=True)


def run_eval(steps, dev, info):
    """evaluate_batch on the padded batch against evaluate_batch_jagged on the packed one, B = 256 geometric histories"""
    pad, _, pk, tgt = batches("geometric", EVAL_B, dev)
    m, _ = make(dev)
    m.eval()
    metrics = torch.zeros(6, device=dev)
    calls = {"padded": lambda: m.evaluate_batch(pad["input_ids"], tgt, metrics),
              "packed": lambda: m.evaluate_batch_jagged(pk["input_ids"], pk["offsets"], pk["max_len"], tgt, metrics)}
    graphs = {k: harness.graphed(f, 3)[0] for k, f in calls.items()}
    times = {"padded": [], "packed": []}
    for _ in range(3):
        for k in times:
            times[k].append(harness.timed(graphs[k].replay, steps, 1)[0])
    out = dict(workload="eval256", B=EVAL_B, packed_tokens=pk["input_ids"].numel(), padded_tokens=pad["input_ids"].numel(), **info)
    for k in times:
        out[k] = dict(call_ms=round(statistics.median(times[k]), 4), runs_ms=[round(t, 4) for t in times[k]])
    out["packed_over_padded"] = round(out["packed"]["call_ms"] / out["padded"]["call_ms"], 4)
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--profile", default="geo1024", help="workloads that also get a per-kernel torch.profiler breakdown")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sasrec_jagged.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    info = harness.card(dev)
    prof = set(args.profile.split(",")) if args.profile else set()
    for name in args.workloads.split(","):
        run(name, args.steps, dev, info, name in prof)
    run_eval(args.steps, dev, info)


if __name__ == "__main__":
    main()
