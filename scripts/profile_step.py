"""Per-kernel device time of one HSTU training step, replayed from a CUDA graph under torch.profiler.

    python scripts/profile_step.py [--config cfg2|cfg3] [--steps K]

Builds the step bench.py times (the same model, optimizer, batch shape and deferred weight gradients), captures it in a graph,
then profiles K replays and prints each kernel's device time per step, grouped by name, with the card's name, power limit and
max SM clock read in the same run.  Kernels on the side stream overlap the main stream, so the column sums to more than the
step's wall time, which is measured separately without the profiler.  With programmatic dependent launch a kernel's CTAs start
once every CTA of the kernel before it has started, so a kernel's time includes its wait for that kernel's last round."""
import argparse
import os
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench  # noqa: E402
from scripts import harness  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2", choices=sorted(bench.CONFIGS))
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    from genrec_b200 import _lib
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatAdam

    dev = torch.device("cuda:0")
    card = harness.card(dev)
    torch.cuda.set_device(dev)
    _lib.ensure_device(dev)
    c = bench.CONFIGS[args.config]
    cfg = dict(c["model"])
    B, L, V = c["batch"], cfg["max_seq_len"], cfg["num_items"]
    torch.manual_seed(0)
    model = HSTU(**cfg).to(dev).train()
    opt = FlatAdam(model, lr=1e-3, betas=(0.9, 0.98), unit_loss_grad=True, defer_weight_grads=True)
    ids, ts, tg = (t.to(dev) for t in bench.synth_batch(B, L, V, 0))

    def step():
        _, loss = model(ids, ts, tg)
        loss.backward()
        opt.step()
        return loss

    graph, _ = harness.graphed(step, 3)
    wall_us = harness.timed(graph.replay, args.steps, 10)[0] * 1e3

    kernels = harness.profile(graph.replay, args.steps, 0)
    total, calls = harness.largest_first(kernels, harness.short_name), defaultdict(int)
    for k, (_, n) in kernels.items():
        calls[harness.short_name(k)] += n
    busy = sum(total.values()) / args.steps

    print(f"card: {card['gpu']}, {card['power_limit_and_max_sm_clock']} (name, power limit, max SM clock)")
    print(f"{args.config}: B={B} L={L} D={cfg['embed_dim']} blocks={cfg['num_blocks']} V={V}; {args.steps} graph replays")
    print(f"step wall time (CUDA events, no profiler): {wall_us:.1f} us; kernel time summed over both streams: {busy:.1f} us")
    print()
    print("| kernel | launches / step | us / step | share of summed kernel time |")
    print("|---|---:|---:|---:|")
    for name, us in total.items():
        per = us / args.steps
        print(f"| `{name}` | {calls[name] / args.steps:g} | {per:.1f} | {100 * per / busy:.1f}% |")


if __name__ == "__main__":
    main()
