"""Training step of HSTU on a packed (jagged) batch against the left-padded batch of the same users.

For each workload one seeded batch of users is drawn as a jagged batch on the device; the padded step trains on collate_jagged of it
and the packed step on pack_jagged of it.  A step is forward, backward and the FlatAdam update (unit_loss_grad, deferred weight
gradients, as bench.py trains), captured in a CUDA graph and replayed.  The two graphs are timed with CUDA events, alternated three
times in one process; the attention kernels' device times come from a separate torch.profiler run of one eager step each.
Dropout is 0, so both steps optimise the same objective: the padded batch's targets at pad inputs (hstu_collate_fn's shift makes the
last pad row predict the first item) are zeroed, and the two losses must agree to rounding.

    python scripts/bench_jagged.py [--steps 20] [--workloads cfg2,d64,short,full]

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

CFG2 = dict(num_items=12101, max_seq_len=200, embed_dim=128, num_heads=4, num_blocks=4)
WORKLOADS = {
    "cfg2": (CFG2, "uniform", "lengths U[50, 200]"),
    "d64": (dict(CFG2, embed_dim=64, num_heads=2, num_blocks=2), "uniform", "lengths U[50, 200], d=64 H=2, 2 blocks"),
    "short": (CFG2, "geometric", "lengths geometric, mean 10, capped at 50"),
    "full": (CFG2, "full", "every length 200"),
}
B = 128


def jagged_batch(kind, V, seed, dev):
    g = torch.Generator().manual_seed(seed)
    if kind == "uniform":
        lens = torch.randint(50, 201, (B,), generator=g)
    elif kind == "full":
        lens = torch.full((B,), 200)
    else:
        lens = harness.geometric_lengths(B, 10, 1, 50, g)
    N = int(lens.sum())
    w = torch.arange(1, V + 1, dtype=torch.float64).pow(-1.1)
    items = torch.multinomial(w, N, replacement=True, generator=g) + 1
    gaps = torch.empty(N).exponential_(1.0 / (3 * 86400.0), generator=g).long() + 1
    ts = 1_300_000_000 + torch.cumsum(gaps, 0)
    tgt = torch.multinomial(w, B, replacement=True, generator=g) + 1
    off = torch.zeros(B + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(lens, 0)
    return items.to(dev), ts.to(dev), off.to(dev), tgt.to(dev)


def make(model_cfg, dev):
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatAdam
    torch.manual_seed(0)
    m = HSTU(dropout=0.0, **model_cfg).to(dev).train()
    opt = FlatAdam(m, lr=1e-3, betas=(0.9, 0.98), unit_loss_grad=True, defer_weight_grads=True)
    return m, opt


ATTENTION_KERNELS = ("hstu_attn", "hstu_bias_index", "hstu_idle_rows")    # the attention, its bias index and the idle-row zeroing


def run(name, steps, dev, info):
    from genrec_b200.data import collate_jagged, pack_jagged
    model_cfg, kind, desc = WORKLOADS[name]
    items, ts, off, tgt = jagged_batch(kind, model_cfg["num_items"], 1234, dev)
    pad = collate_jagged(items, off, tgt, model_cfg["max_seq_len"], timestamps=ts)
    pad_tg = torch.where(pad["input_ids"] == 0, 0, pad["targets"])
    pk = pack_jagged(items, off, tgt, model_cfg["max_seq_len"], timestamps=ts)
    T, L = pk["input_ids"].numel(), pad["input_ids"].shape[1]

    res = {}
    for path in ("padded", "packed"):
        m, opt = make(model_cfg, dev)

        def step(m=m, opt=opt, path=path):
            if path == "padded":
                _, loss = m(pad["input_ids"], pad["timestamps"], pad_tg)
            else:
                _, loss = m.forward_jagged(pk["input_ids"], pk["offsets"], pk["max_len"], pk["timestamps"], pk["targets"])
            loss.backward()
            opt.step()
            return loss

        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()           # step_peak_mem_mb: the step's working memory above the resident model, batch
                                                       # and the other path's buffers
        torch.cuda.reset_peak_memory_stats()
        loss0 = step().item()                          # the first step's loss, from the same initial parameters on both paths
        g, _ = harness.graphed(step, 3)
        g.replay()
        torch.cuda.synchronize()
        res[path] = dict(model=m, opt=opt, step=step, graph=g, loss0=loss0, peak_mb=(torch.cuda.max_memory_allocated() - base) / 2 ** 20)
    times = {"padded": [], "packed": []}
    for _ in range(3):
        for path in ("padded", "packed"):
            times[path].append(harness.timed(res[path]["graph"].replay, steps, 1)[0])
    out = dict(workload=name, desc=desc, B=B, **{k: model_cfg[k] for k in ("embed_dim", "num_heads", "num_blocks", "num_items")},
               padded_L=L, padded_tokens=B * L, packed_tokens=T, padding_share=round(1 - T / (B * L), 4), **info)
    for path in ("padded", "packed"):
        ms = statistics.median(times[path])
        out[path] = dict(step_ms=round(ms, 4), runs_ms=[round(t, 4) for t in times[path]], seq_per_s=round(B / ms * 1e3, 1),
                         step_peak_mem_mb=round(res[path]["peak_mb"], 1), loss_step1=res[path]["loss0"])
    out["packed_over_padded"] = round(out["packed"]["step_ms"] / out["padded"]["step_ms"], 4)
    out["loss_rel_diff"] = abs(res["packed"]["loss0"] - res["padded"]["loss0"]) / abs(res["padded"]["loss0"])
    for path in ("padded", "packed"):
        res[path]["graph"].reset()
        attn = {k: v for k, v in harness.profile(res[path]["step"]).items() if any(part in k for part in ATTENTION_KERNELS)}
        attn = harness.largest_first(attn, lambda k: harness.short_name(k, "<"))
        out[path]["attention_kernels_us"] = {k: round(us, 1) for k, us in attn.items()}
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jagged.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    info = harness.card(dev)
    for name in args.workloads.split(","):
        run(name, args.steps, dev, info)


if __name__ == "__main__":
    main()
