"""Per-kernel device time of one HSTU training step, replayed from a CUDA graph under torch.profiler.

    python scripts/profile_step.py [--config cfg2|cfg3] [--steps K]

Builds the step bench.py times (the same model, optimizer, batch shape and deferred weight gradients), captures it in a graph,
then profiles K replays and prints each kernel's device time per step, grouped by name, with the card's name, power limit and
max SM clock read in the same run.  Kernels on the side stream overlap the main stream, so the column sums to more than the
step's wall time, which is measured separately without the profiler.  With programmatic dependent launch a kernel's CTAs start
once every CTA of the kernel before it has started, so a kernel's time includes its wait for that kernel's last round."""
import argparse
import os
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import bench  # noqa: E402


def short_name(name):
    name = name.split("(")[0] if not name.startswith("void ") else name[5:].split("(")[0]
    return name.replace("grb::", "")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="cfg2", choices=sorted(bench.CONFIGS))
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    from genrec_b200 import _lib
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatAdam

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    dev = torch.device("cuda:0")
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

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            step()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        step()
    for _ in range(10):
        graph.replay()
    torch.cuda.synchronize()

    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.steps):
        graph.replay()
    t1.record()
    torch.cuda.synchronize()
    wall_us = t0.elapsed_time(t1) * 1e3 / args.steps

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            graph.replay()
        torch.cuda.synchronize()
    total, calls = defaultdict(float), defaultdict(int)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            total[short_name(e.name)] += e.time_range.elapsed_us()
            calls[short_name(e.name)] += 1
    busy = sum(total.values()) / args.steps

    print(f"card: {'; '.join(card)} (name, power limit, max SM clock)")
    print(f"{args.config}: B={B} L={L} D={cfg['embed_dim']} blocks={cfg['num_blocks']} V={V}; {args.steps} graph replays")
    print(f"step wall time (CUDA events, no profiler): {wall_us:.1f} us; kernel time summed over both streams: {busy:.1f} us")
    print()
    print("| kernel | launches / step | us / step | share of summed kernel time |")
    print("|---|---:|---:|---:|")
    for name, us in sorted(total.items(), key=lambda kv: -kv[1]):
        per = us / args.steps
        print(f"| `{name}` | {calls[name] / args.steps:g} | {per:.1f} | {100 * per / busy:.1f}% |")


if __name__ == "__main__":
    main()
