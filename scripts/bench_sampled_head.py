"""Measure the sampled-softmax head on the GPU: python scripts/bench_sampled_head.py [--out result.json]

  1. head alone at T = 128 x 200 tokens, D = 128 and 64: the full head at C = 12,102 next to the sampled head at N = 128, 1,024 and
     4,096, alternated in one session, each call replayed from a CUDA graph and timed with CUDA events; the sampled head again at
     C = 1,000,001 (its time must not depend on C);
  2. the time of each kernel of the sampled head (torch.profiler, a run of its own), and for the row pass the least time the
     hardware could take: the larger of 6 T D (N + 1) FLOP at 989 TFLOP/s and the bytes it must move at 3.35 TB/s (data-sheet
     figures of the H100 SXM at 700 W);
  3. one training step of HSTU at the cfg2 geometry with V = 1,000,000 and 10,000,000 items and N = 1,024 under FlatAdam, dense and
     with lazy_table=True alternated, and the optimizer's part of it (the dense table is nearly all the parameters); the lazy
     kernels' times under torch.profiler and the lazy table pass against its byte bound (34 B per touched element at 3.35 TB/s).
     --skip-head runs this part only.
A GPU is required; there is no fallback.  The card's name and power limit are read in the same run and printed with the numbers."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts import harness  # noqa: E402

PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12
EPS = 1e-5


def graph_time(fn, iters=20, rounds=5):
    """median over `rounds` of the mean time (ms) of `iters` replays of fn captured in a CUDA graph"""
    graph, _ = harness.graphed(fn, 3)
    graph.replay()
    return statistics.median(harness.timed(graph.replay, iters, 0)[0] for _ in range(rounds))


class Head:
    """operands of one head call at (T, D, C) and closures that run the full / the sampled head through the C ABI"""

    def __init__(self, T, D, C, dev):
        from genrec_b200 import functional as Fn
        g = torch.Generator(device=dev).manual_seed(T + D + C)
        self.T, self.D, self.C, self.dev = T, D, C, dev
        self.x = torch.randn(T, D, device=dev, generator=g)
        self.ln_g, self.ln_b = torch.ones(D, device=dev), torch.zeros(D, device=dev)
        self.tb = Fn.cast_bf16(0.05 * torch.randn(C, D, device=dev, generator=g))
        self.tg = torch.randint(1, C, (T,), device=dev, generator=g)
        self.log_q = torch.log_softmax(torch.randn(C, device=dev, generator=g), 0)
        self.dx, self.dE = torch.empty_like(self.x), torch.zeros(C, D, device=dev)
        self.dg, self.db = torch.zeros(D, device=dev), torch.zeros(D, device=dev)
        self.loss = torch.empty((), device=dev)
        self.gen = g

    def full(self):
        from genrec_b200 import _lib
        from genrec_b200._lib import check, ptr, stream_ptr
        lib = _lib.load()
        ws = torch.empty(lib.grb_head_workspace_bytes(self.T, self.D, self.C), dtype=torch.uint8, device=self.dev)
        return lambda: check(lib.grb_head_loss_forward_backward(ptr(self.x), ptr(self.ln_g), ptr(self.ln_b), EPS, ptr(self.tb), ptr(self.tg), self.T,
                                                                self.D, self.C, ptr(self.loss), ptr(self.dx), ptr(self.dE), ptr(self.dg), ptr(self.db),
                                                                ptr(ws), stream_ptr(self.dev)))

    def sampled(self, N):
        from genrec_b200 import _lib
        from genrec_b200._lib import check, ptr, stream_ptr
        lib = _lib.load()
        neg = torch.randint(1, self.C, (N,), device=self.dev, generator=self.gen)
        ws = torch.empty(lib.grb_head_sampled_workspace_bytes(self.T, self.D, N), dtype=torch.uint8, device=self.dev)
        return lambda: check(lib.grb_head_sampled_loss_forward_backward(ptr(self.x), ptr(self.ln_g), ptr(self.ln_b), EPS, ptr(self.tb), ptr(self.tg),
                                                                        ptr(neg), ptr(self.log_q), self.T, self.D, self.C, N, ptr(self.loss),
                                                                        ptr(self.dx), ptr(self.dE), ptr(self.dg), ptr(self.db), ptr(ws),
                                                                        stream_ptr(self.dev)))


def head_alone(dev, T, res):
    for D in (128, 64):
        small, big = Head(T, D, 12102, dev), Head(T, D, 1_000_001, dev)
        runs = [("full head C=12102", small.full())]
        for N in (128, 1024, 4096):
            runs.append((f"sampled N={N} C=12102", small.sampled(N)))
        runs.append(("sampled N=1024 C=1000001", big.sampled(1024)))
        times = {k: [] for k, _ in runs}
        for _ in range(3):                               # alternate the variants: drift of the card hits all of them alike
            for k, fn in runs:
                times[k].append(graph_time(fn, rounds=3))
        for k, v in times.items():
            res[f"head D={D} T={T} {k} ms"] = round(statistics.median(v), 4)
        del small, big
        torch.cuda.empty_cache()


def per_kernel(dev, T, res):
    D = 128
    h = Head(T, D, 12102, dev)
    for N in (1024, 4096):
        reps = 20
        kernels = harness.profile(h.sampled(N), reps, 3)
        for name, (t, _) in kernels.items():
            for short in ("sce_gather_kernel", "sce_target_kernel", "sce_rows_kernel", "sce_table_kernel", "sce_scatter_kernel", "ln_fwd_kernel",
                          "ln_bwd_kernel"):
                if short in name:
                    res[f"kernel D={D} T={T} N={N} {short} us"] = round(t / reps, 2)
        Npad = (N + 63) // 64 * 64
        flop_t = 6.0 * T * D * (N + 1) / PEAK_FLOPS
        bytes_t = (T * D * 2 + T * D * 4 + Npad * D * 2 + T * 8 * 4) / PEAK_BYTES      # H in, dH out, Es once, the per-token vectors
        res[f"row pass bound D={D} T={T} N={N} us"] = round(max(flop_t, bytes_t) * 1e6, 2)
        res[f"row pass bound D={D} T={T} N={N} binds"] = "FLOP at 989 TFLOP/s" if flop_t >= bytes_t else "bytes at 3.35 TB/s"


class _DenseMode:
    """Run `opt` (built with lazy_table=True) as the dense FlatAdam while a graph is captured: the step takes the dense path and the
    forwards mark no rows.  Both variants then share one model and one set of flat buffers (23 GB at V = 10,000,000)."""

    def __init__(self, model, opt, on):
        self.model, self.opt, self.on = model, opt, on

    def __enter__(self):
        if self.on:
            self.opt.lazy_table, self.model._row_marker = False, None

    def __exit__(self, *exc):
        if self.on:
            self.opt.lazy_table, self.model._row_marker = True, self.opt


def graph_time_alternating(variants, iters=5, rounds=3, alternations=3):
    """{name: (fn, dense?)} -> {name: median ms}, the variants alternated `alternations` times in one session"""
    times = {k: [] for k in variants}
    for _ in range(alternations):
        for k, (fn, ctx) in variants.items():
            with ctx:
                times[k].append(graph_time(fn, iters=iters, rounds=rounds))
    return {k: statistics.median(v) for k, v in times.items()}


def full_step(dev, res, V):
    """One cfg2-geometry HSTU training step with N = 1,024 sampled negatives, and FlatAdam's part of it (the marks of the step's ids
    and the optimizer step), dense against lazy_table=True, alternated; then the lazy kernels under torch.profiler."""
    from genrec_b200.data import sample_negatives
    from genrec_b200.hstu import HSTU
    from genrec_b200.optim import FlatAdam
    B, L, N, D = 128, 200, 1024, 128
    torch.manual_seed(0)
    with torch.device(dev):          # a 10 M-row table is initialised on the GPU, not on the CPU
        model = HSTU(num_items=V, max_seq_len=L, embed_dim=D, num_heads=4, num_blocks=4, dropout=0.2).train()
    opt = FlatAdam(model, lr=1e-3, betas=(0.9, 0.98), unit_loss_grad=True, lazy_table=True)
    g = torch.Generator(device=dev).manual_seed(1)
    ids = torch.randint(1, V + 1, (B, L), device=dev, generator=g)
    tg = torch.randint(1, V + 1, (B, L), device=dev, generator=g)
    ts = 1_300_000_000 + torch.cumsum(torch.randint(1, 86400, (B, L), device=dev, generator=g), 1)
    neg = torch.empty(N, dtype=torch.int64, device=dev)

    def step():
        neg.copy_(sample_negatives(V, N, device=dev)[0])       # redrawn on the device inside the captured step
        _, loss = model(ids, ts, tg, negatives=neg)
        loss.backward()
        opt.step()

    def optimizer_part():
        if opt.lazy_table:           # what the forwards add to the optimizer's work: the marks of the step's ids
            opt._mark(ids); opt._mark(tg); opt._mark(neg)
        opt.step()

    t = graph_time_alternating({"dense step": (step, _DenseMode(model, opt, True)), "lazy step": (step, _DenseMode(model, opt, False)),
                                "dense opt": (optimizer_part, _DenseMode(model, opt, True)),
                                "lazy opt": (optimizer_part, _DenseMode(model, opt, False))})
    res[f"cfg2 geometry V={V} N={N} training step ms, dense FlatAdam"] = round(t["dense step"], 3)
    res[f"cfg2 geometry V={V} N={N} training step ms, lazy_table=True"] = round(t["lazy step"], 3)
    res[f"cfg2 geometry V={V} FlatAdam step alone ms, dense"] = round(t["dense opt"], 3)
    res[f"cfg2 geometry V={V} FlatAdam marks + step ms, lazy_table=True"] = round(t["lazy opt"], 3)
    table = model.item_embedding.weight.numel()
    res[f"V={V} table share of the parameters"] = round(table / sum(p.numel() for p in model.parameters()), 4)

    reps, touched = 5, []

    def marked_step():
        opt._mark(ids); opt._mark(tg); opt._mark(neg)
        touched.append(opt._row_count[0].clone())
        opt.step()

    kernels = harness.profile(marked_step, reps, 0)
    rows = int(touched[0])
    res[f"V={V} touched rows per step"] = rows
    for name, (t_us, _) in kernels.items():
        for short in ("rowset_mark_kernel", "lazy_table_step_kernel", "adam_step_kernel", "rowset_reset_kernel", "adam_tick_kernel"):
            if short in name:
                res[f"V={V} kernel {short} us per step"] = round(t_us / reps, 2)
    bound_us = 34.0 * rows * D / PEAK_BYTES * 1e6
    res[f"V={V} lazy table pass byte bound us (34 B per touched element at 3.35 TB/s)"] = round(bound_us, 2)
    k = res.get(f"V={V} kernel lazy_table_step_kernel us per step")
    if k:
        res[f"V={V} lazy table pass share of its byte bound"] = round(bound_us / k, 3)
    del model, opt
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--skip-head", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sampled_head.py needs a CUDA GPU (sm_90a); there is no fallback")
    from genrec_b200 import _lib
    dev = torch.device("cuda:0")
    _lib.ensure_device(dev)
    res = harness.card(dev)
    T = 128 * 200
    if not args.skip_head:
        head_alone(dev, T, res)
        per_kernel(dev, T, res)
    if not args.skip_step:
        for V in (1_000_000, 10_000_000):
            full_step(dev, res, V)
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
