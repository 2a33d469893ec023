"""Stand-alone device timings of the secondary kernels (RQ-VAE residual argmin, SASRec attention, HSTU layer at cfg-3 geometry,
cached incremental HSTU inference next to full recompute, RQ-VAE Sinkhorn and k-means init) with CUDA events, against the relevant
roofline or the torch code they replace.  Prints one JSON line per measurement; `bench_kernels.py rqvae_train` runs only the RQ-VAE
training rows, `bench_kernels.py linear_bwd` only the linear-backward and SASRec training-step rows, `bench_kernels.py head_topk` only
the fused top-k head rows, `bench_kernels.py tiger` only the TIGER rows (training step, generate eager / graph / uncached loop, wide beams),
`bench_kernels.py hstu_attn` only the HSTU attention backward rows, `bench_kernels.py head_rank` only the rows of evaluation without
logits, `bench_kernels.py head_candidates` only the rows of retrieval without logits."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import genrec_b200.functional as Fn
from genrec_b200.hstu import HSTULayer
from scripts import harness


def graph_ms(fn, reps=10, iters=10):
    """Device time (ms) per call with `reps` calls captured in one CUDA graph (no host gaps: what a small kernel really costs)."""
    graph, _ = harness.graphed(fn, 3, calls=reps)
    return harness.timed(graph.replay, iters, 1)[0] / reps


def peak_mb(fn):
    """MiB allocated at the peak of one call of fn, above what was allocated before it, after one untimed call"""
    fn()
    base = torch.cuda.memory_allocated()
    return (harness.peak(fn) - base) / 2 ** 20


def bench_extend(dev):
    """Cached incremental inference (HSTU.extend) next to full recompute (HSTU.last_logits) on the same full sequences: one new
    item per user on a history of L - 1, and the prefill of the whole history (extend on an empty state).  Both graph-captured.
    The state is rewound on the device before every call (lengths.fill_, one small kernel inside the timed graph), so every call
    appends at the same position.  The chunk-attention kernel's bytes are the cache K | V and timestamps it must read."""
    from genrec_b200.hstu import HSTU
    info = harness.card(dev)
    HBM = 3.35e12   # H100 SXM data sheet, bytes/s
    geoms = (("cfg2", dict(num_items=12101, embed_dim=128, num_heads=4, num_blocks=4), 200, (1, 128)),
             ("cfg3", dict(num_items=12101, embed_dim=256, num_heads=8, num_blocks=8), 2048, (1, 32)))
    g = torch.Generator().manual_seed(0)
    for name, geo, L, batches in geoms:
        torch.manual_seed(0)
        m = HSTU(max_seq_len=L, dropout=0.0, **geo).to(dev).eval()
        D, NB = geo["embed_dim"], geo["num_blocks"]
        for B in batches:
            ids = torch.randint(1, geo["num_items"] + 1, (B, L), generator=g).to(dev)
            ts = (1_300_000_000 + torch.cumsum(torch.randint(1, 3 * 86400, (B, L), generator=g), 1)).to(dev)
            st = m.new_state(B, L)
            m.extend(st, ids[:, :-1], ts[:, :-1])

            def one():
                st.lengths.fill_(L - 1)
                st.items_bound = L - 1
                return m.extend(st, ids[:, -1:], ts[:, -1:])

            def prefill():
                st.lengths.zero_()
                st.items_bound = 0
                return m.extend(st, ids, ts)

            full_ms = graph_ms(lambda: m.last_logits(ids, ts))
            for work, fn, keys in (("extend_1", one, L), ("prefill", prefill, None)):
                ms = graph_ms(fn)
                row = dict(kernel="hstu_extend", geometry=name, workload=work, B=B, history=L - 1 if work == "extend_1" else 0,
                           new_items=1 if work == "extend_1" else L, extend_us=ms * 1e3, last_logits_us=full_ms * 1e3,
                           speedup_vs_last_logits=full_ms / ms, **info)
                if keys is not None:
                    attn_us = harness.mean_launch_us(harness.profile(fn, 20), "hstu_attn_extend_kernel")
                    byt = B * keys * (2 * D * 2 + 8)            # per layer: K | V bf16 + int64 timestamp of every cached key
                    row.update(attn_kernel_us=attn_us, attn_bytes_per_layer=byt, attn_hbm_gbs=byt / attn_us / 1e3,
                               attn_frac_of_hbm_peak=byt / (attn_us * 1e-6) / HBM, blocks=NB)
                print(json.dumps(row), flush=True)
            assert torch.isfinite(one()).all()


POOL_GEOMS = (("cfg2", dict(num_items=12101, embed_dim=128, num_heads=4, num_blocks=4), 4096, 200, 128, True),
              ("cfg3", dict(num_items=12101, embed_dim=256, num_heads=8, num_blocks=8), 512, 2048, 32, False))


def _pool_workload(dev, name, geo, nusers, cap, B):
    """A pool of `nusers` users with seeded history lengths (none a multiple of the page size) and B random users to extend by one
    item -> (model, pool, lens, hist, hts, users, one(**kw)); one() rewinds the users' lengths on the device and calls
    extend_users(..., **kw)."""
    from genrec_b200.hstu import HSTU
    g = torch.Generator().manual_seed(1)
    torch.manual_seed(0)
    m = HSTU(max_seq_len=cap, dropout=0.0, **geo).to(dev).eval()
    ps = 64
    lens = torch.randint(1, cap, (nusers,), generator=g)
    lens[lens % ps == 0] -= 1                                  # the timed item stays inside the user's last page
    pool = m.new_pool(max_users=nusers, num_pages=int(((lens + ps) // ps).sum()), page_size=ps, max_items=cap)
    hist = torch.randint(1, geo["num_items"] + 1, (nusers, cap), generator=g)
    hts = 1_300_000_000 + torch.cumsum(torch.randint(1, 3 * 86400, (nusers, cap), generator=g), 1)
    pad = torch.arange(cap)[None, :] < (cap - 1 - lens)[:, None]   # user u: lens[u] items, then the timed one in column cap-1
    hist[pad] = 0
    hts[pad] = 0
    chunk = 128 if name == "cfg2" else 16
    for u0 in range(0, nusers, chunk):                         # device users: pages follow the real lengths, not the host bound
        us = torch.arange(u0, min(u0 + chunk, nusers))
        m.extend_users(pool, us.to(dev), hist[us, :-1].to(dev), hts[us, :-1].to(dev))
    assert not pool.overflowed().any()
    users = torch.randperm(nusers, generator=g)[:B]
    users_dev = users.to(dev)
    ulens = lens[users].to(dev, torch.int32)
    ids1, ts1 = hist[users, -1:].to(dev), hts[users, -1:].to(dev)

    def one(**kw):
        pool.lengths.index_copy_(0, users_dev, ulens)
        return m.extend_users(pool, users_dev, ids1, ts1, **kw)

    return m, pool, lens, hist, hts, users, one


def bench_head_topk(dev):
    """The fused top-k head (Fn.head_topk: LayerNorm, wgmma scoring with per-row lists, merge) against the logits path it replaces
    for serving (Fn.head_logits, column 0 set to -inf, torch.topk), both graph-captured, k = 10 and 64: the head alone at the project's
    catalog (cfg2: D = 128, C = 12,102) and at a 1,000,000-item catalog, then extend_users(top_k=10) against extend_users + the same
    top-k on the cfg2 pool workload.  The scoring kernel's time (torch.profiler) is set against its bound, the larger of the table
    read (C D 2 bytes at 3.35 TB/s) and the GEMM (2 R C D FLOP at 989 TFLOP/s), both H100 SXM data-sheet figures."""
    info = harness.card(dev)
    HBM, BF16 = 3.35e12, 989e12
    g = torch.Generator().manual_seed(0)
    D, eps = 128, 1e-5
    for C, batches in ((12102, (1, 128)), (1000001, (1, 128, 1024))):
        tb = (0.05 * torch.randn(C, D, generator=g)).to(torch.bfloat16).to(dev)
        ln_g, ln_b = (1 + 0.1 * torch.randn(D, generator=g)).to(dev), (0.1 * torch.randn(D, generator=g)).to(dev)
        for B in batches:
            x = torch.randn(B, D, generator=g).to(dev)
            for k in (10, 64):
                def fused():
                    return Fn.head_topk(x, ln_g, ln_b, tb, eps, k)

                def logits_topk():
                    lo = Fn.head_logits(x[:, None, :], ln_g, ln_b, tb, tb, eps)[:, 0, :]
                    lo[:, 0] = float("-inf")
                    return torch.topk(lo, k, dim=1)

                assert torch.equal(fused().scores, logits_topk().values)
                f_ms, b_ms = graph_ms(fused), graph_ms(logits_topk)
                kern = harness.mean_launch_us(harness.profile(fused, 20), "head_topk_kernel")
                t_bytes, t_flop = C * D * 2 / HBM * 1e6, 2 * B * C * D / BF16 * 1e6
                bound = max(t_bytes, t_flop)
                print(json.dumps(dict(kernel="head_topk", workload="head", D=D, C=C, B=B, k=k, fused_us=f_ms * 1e3,
                                      logits_topk_us=b_ms * 1e3, speedup_vs_logits_topk=b_ms / f_ms, scoring_kernel_us=kern,
                                      bound_us=bound, bound_by="table read" if t_bytes >= t_flop else "bf16 GEMM",
                                      fused_over_bound=f_ms * 1e3 / bound, scoring_kernel_over_bound=kern / bound, **info)), flush=True)
        del tb
        torch.cuda.empty_cache()
    name, geo, nusers, cap, B, _ = POOL_GEOMS[0]
    m, pool, lens, hist, hts, users, one = _pool_workload(dev, name, geo, nusers, cap, B)

    def one_topk():
        lo = one()
        lo[:, 0] = float("-inf")
        return torch.topk(lo, 10, dim=1)

    assert torch.equal(one(top_k=10).scores, one_topk().values)
    f_ms, b_ms = graph_ms(lambda: one(top_k=10)), graph_ms(one_topk)
    print(json.dumps(dict(kernel="head_topk", workload="extend_users", geometry=name, pool_users=nusers, B=B, k=10, max_items=cap,
                          fused_us=f_ms * 1e3, logits_topk_us=b_ms * 1e3, speedup_vs_logits_topk=b_ms / f_ms, **info)), flush=True)


def bench_head_candidates(dev):
    """Retrieval without logits (Fn.head_candidates: LayerNorm, bound sweep, threshold, collect sweep, overflow passes, sort)
    against the logits path (Fn.head_logits, column 0 set to -inf, torch.topk), both graph-captured, at D = 128: C = 12,102 and
    1,000,001, B = 1, 128 and 1,024, k = 64 (the top-k head), 256, 1,024 and 2,048.  Then a clustered table whose best 3,000 items
    sit in one item range for every row, the per-kernel times (torch.profiler, a run of their own) and extend_users(num_candidates=
    500) on the cfg2 pool workload against extend_users + torch.topk.  The one-sweep bound is the larger of the table read (C D 2
    bytes at 3.35 TB/s) and the GEMM (2 B C D FLOP at 989 TFLOP/s), H100 SXM data-sheet figures; peak memory is
    torch.cuda.max_memory_allocated above the inputs."""
    info = harness.card(dev)
    HBM, BF16 = 3.35e12, 989e12
    D, eps = 128, 1e-5
    gd = torch.Generator(device=dev).manual_seed(0)

    def measure(workload, x, ln_g, ln_b, tb, k, profile_kernels):
        B, C = x.shape[0], tb.shape[0]

        def fused():
            return Fn.head_candidates(x, ln_g, ln_b, tb, eps, k)

        def logits_topk():
            lo = Fn.head_logits(x[:, None, :], ln_g, ln_b, tb, tb, eps)[:, 0, :]
            lo[:, 0] = float("-inf")
            return torch.topk(lo, k, dim=1)

        assert torch.equal(fused().scores, logits_topk().values)
        f_ms = graph_ms(fused)
        b_ms = graph_ms(logits_topk, reps=2, iters=5)
        t_bytes, t_flop = C * D * 2 / HBM * 1e6, 2 * B * C * D / BF16 * 1e6
        bound = max(t_bytes, t_flop)
        row = dict(kernel="head_candidates", workload=workload, D=D, C=C, B=B, k=k, fused_us=f_ms * 1e3, logits_topk_us=b_ms * 1e3,
                   speedup_vs_logits_topk=b_ms / f_ms, bound_us=bound, bound_by="table read" if t_bytes >= t_flop else "bf16 GEMM",
                   fused_over_bound=f_ms * 1e3 / bound, fused_peak_mb=peak_mb(fused), logits_topk_peak_mb=peak_mb(logits_topk))
        if profile_kernels:
            prefix = "head_" if k <= 64 else "head_cand"
            kernels = harness.profile(fused, 20)
            row.update(kernels_us={name.split("(")[0][:80]: us / 20 for name, (us, _) in kernels.items() if prefix in name})
        print(json.dumps(dict(**row, **info)), flush=True)

    for C in (12102, 1000001):
        tb = (0.05 * torch.randn(C, D, device=dev, generator=gd)).to(torch.bfloat16)
        ln_g, ln_b = 1 + 0.1 * torch.randn(D, device=dev, generator=gd), 0.1 * torch.randn(D, device=dev, generator=gd)
        for B in (1, 128, 1024):
            x = torch.randn(B, D, device=dev, generator=gd)
            for k in (64, 256, 1024, 2048):
                measure("head", x, ln_g, ln_b, tb, k, profile_kernels=k in (64, 1024))
            del x
            torch.cuda.empty_cache()
        del tb
        torch.cuda.empty_cache()
    # clustered: rows lo .. lo + 2,999 of the table score above every other item for every row of x
    C, B, n = 1000001, 128, 3000
    b = torch.randn(D, device=dev, generator=gd)
    ln_g, ln_b = torch.full((D,), 0.1, device=dev), b
    tb = 0.05 * torch.randn(C, D, device=dev, generator=gd)
    lo = 128 * 70
    tb[lo:lo + n] += 0.05 * b
    tb = tb.to(torch.bfloat16)
    x = torch.randn(B, D, device=dev, generator=gd)
    for k in (500, 1024, 2048):
        measure("clustered", x, ln_g, ln_b, tb, k, profile_kernels=True)
    del tb
    torch.cuda.empty_cache()
    name, geo, nusers, cap, B, _ = POOL_GEOMS[0]
    m, pool, lens, hist, hts, users, one = _pool_workload(dev, name, geo, nusers, cap, B)

    def one_topk():
        lo = one()
        lo[:, 0] = float("-inf")
        return torch.topk(lo, 500, dim=1)

    assert torch.equal(one(num_candidates=500).scores, one_topk().values)
    runs = {"num_candidates": [], "logits_topk": []}
    for _ in range(3):
        runs["num_candidates"].append(graph_ms(lambda: one(num_candidates=500)) * 1e3)
        runs["logits_topk"].append(graph_ms(one_topk) * 1e3)
    print(json.dumps(dict(kernel="head_candidates", workload="extend_users", geometry=name, pool_users=nusers, B=B, k=500, max_items=cap,
                          us=runs, **info)), flush=True)


LOGITS_CAP_GB = 16


def bench_head_rank(dev):
    """Leave-one-out evaluation without logits (Fn.head_rank_metrics: LayerNorm, target gather and score, wgmma sweep counting the
    target's rank, finish) against the logits path it replaces (Fn.head_logits on the last rows + Fn.eval_rank_metrics), both
    graph-captured, at D = 128.  The logits path runs only where its [B, C] fp32 logits fit under LOGITS_CAP_GB.  The sweep kernel's
    time (torch.profiler) is set against its bound, the larger of the table read (C D 2 bytes at 3.35 TB/s) and the GEMM (2 B C D
    FLOP at 989 TFLOP/s), both H100 SXM data-sheet figures.  Peak memory is torch.cuda.max_memory_allocated above the inputs.  Last,
    HSTU.evaluate_batch at the cfg2 geometry, B = 128, against eval_rank_metrics(last_logits(...)), alternated three times."""
    from genrec_b200.hstu import HSTU
    info = harness.card(dev)
    HBM, BF16 = 3.35e12, 989e12
    D, eps = 128, 1e-5
    gd = torch.Generator(device=dev).manual_seed(0)

    for C in (12102, 1000001, 10000001):
        tb = (0.05 * torch.randn(C, D, device=dev, generator=gd)).to(torch.bfloat16)
        ln_g, ln_b = 1 + 0.1 * torch.randn(D, device=dev, generator=gd), 0.1 * torch.randn(D, device=dev, generator=gd)
        for B in (128, 1024):
            x = torch.randn(B, D, device=dev, generator=gd)
            tg = torch.randint(1, C, (B,), device=dev, generator=gd)
            met = torch.zeros(6, device=dev)

            def fused():
                return Fn.head_rank_metrics(x, ln_g, ln_b, tb, eps, tg, met)

            def logits_path():
                return Fn.eval_rank_metrics(Fn.head_logits(x[:, None, :], ln_g, ln_b, tb, tb, eps)[:, 0, :], tg, met)

            logits_gb = B * C * 4 / 1e9
            t_bytes, t_flop = C * D * 2 / HBM * 1e6, 2 * B * C * D / BF16 * 1e6
            bound = max(t_bytes, t_flop)
            f_ms = graph_ms(fused)
            kern = harness.mean_launch_us(harness.profile(fused, 20), "head_rank_kernel")
            row = dict(kernel="head_rank", D=D, C=C, B=B, fused_us=f_ms * 1e3, kernel_us=kern, bound_us=bound,
                       bound_by="table read" if t_bytes >= t_flop else "bf16 GEMM", kernel_over_bound=kern / bound,
                       fused_peak_mb=peak_mb(fused), logits_gb=logits_gb)
            if logits_gb <= LOGITS_CAP_GB:
                r_f = Fn.head_rank_metrics(x, ln_g, ln_b, tb, eps, tg, want_ranks=True)[1]
                r_l = Fn.eval_rank_metrics(Fn.head_logits(x[:, None, :], ln_g, ln_b, tb, tb, eps)[:, 0, :], tg, want_ranks=True)[1]
                assert torch.equal(r_f, r_l)
                b_ms = graph_ms(logits_path, reps=2, iters=5)
                row.update(logits_path_us=b_ms * 1e3, speedup_vs_logits=b_ms / f_ms, logits_peak_mb=peak_mb(logits_path))
            else:
                row.update(logits_path=f"not run ({logits_gb:.1f} GB of logits, cap {LOGITS_CAP_GB} GB)")
            print(json.dumps(dict(**row, **info)), flush=True)
            del x
            torch.cuda.empty_cache()
        del tb
        torch.cuda.empty_cache()
    # whole evaluate_batch at cfg2 (num_items = 12,101, D = 128, 4 heads, 4 blocks, L = 200), B = 128
    torch.manual_seed(0)
    V, L, B = 12101, 200, 128
    m = HSTU(V, L, 128, 4, 4, dropout=0.0).to(dev).eval()
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(1, V + 1, (B, L), generator=g).to(dev)
    ts = (1_300_000_000 + torch.cumsum(torch.randint(1, 3 * 86400, (B, L), generator=g), 1)).to(dev)
    tg = torch.randint(1, V + 1, (B,), generator=g).to(dev)
    met = torch.zeros(6, device=dev)
    new = lambda: m.evaluate_batch(ids, ts, tg, met)                                     # noqa: E731
    old = lambda: Fn.eval_rank_metrics(m.last_logits(ids, ts), tg, met)                   # noqa: E731
    assert torch.equal(Fn.eval_rank_metrics(m.last_logits(ids, ts), tg)[:3], m.evaluate_batch(ids, ts, tg)[:3])
    runs = {"evaluate_batch": [], "last_logits_eval_rank": []}
    for _ in range(3):
        runs["evaluate_batch"].append(graph_ms(new) * 1e3)
        runs["last_logits_eval_rank"].append(graph_ms(old) * 1e3)
    print(json.dumps(dict(kernel="head_rank", workload="HSTU.evaluate_batch", geometry="cfg2", B=B, L=L, C=V + 1, us=runs,
                          peak_mb=dict(evaluate_batch=peak_mb(new), last_logits_eval_rank=peak_mb(old)), **info)), flush=True)


def bench_pool(dev):
    """Serving from the paged pool (HSTU.extend_users): a pool of many users with seeded history lengths, one new item for a random
    subset of them, next to the dense HSTUState extend of the same users (cfg2) and last_logits on their left-padded histories.
    Graph-captured with the users as a device tensor.  Every length is a non-multiple of the page size, so the timed item never
    takes a page, and the lengths are rewound on the device before every call (one small kernel inside the timed graph).  The
    allocation kernel and the chunk-attention kernel are timed on their own with torch.profiler."""
    info = harness.card(dev)
    HBM = 3.35e12
    for name, geo, nusers, cap, B, dense in POOL_GEOMS:
        m, pool, lens, hist, hts, users, one = _pool_workload(dev, name, geo, nusers, cap, B)
        D, NB, ps = geo["embed_dim"], geo["num_blocks"], pool.page_size
        ulens = lens[users].to(dev, torch.int32)
        ids1, ts1 = hist[users, -1:].to(dev), hts[users, -1:].to(dev)
        ms = graph_ms(one)
        hist_u, hts_u = hist[users].to(dev), hts[users].to(dev)
        full_ms = graph_ms(lambda: m.last_logits(hist_u, hts_u))
        kernels = harness.profile(one, 20)
        attn_us = harness.mean_launch_us(kernels, "hstu_attn_extend_kernel")
        alloc_us = harness.mean_launch_us(kernels, "hstu_pool_alloc_kernel")
        item = NB * 2 * D * 2 + 8                                   # cached bytes per item: K | V of every block + timestamp
        byt = int((lens[users] + 1).sum()) * (2 * D * 2 + 8)        # per layer: the keys the attention reads
        pages = int(((lens[users] + ps) // ps).sum())
        row = dict(kernel="hstu_pool_extend", geometry=name, workload="extend_1", pool_users=nusers, B=B, page_size=ps, max_items=cap,
                   mean_history=float(lens[users].float().mean()), extend_users_us=ms * 1e3, last_logits_us=full_ms * 1e3,
                   attn_kernel_us=attn_us, alloc_kernel_us=alloc_us, attn_bytes_per_layer=byt, attn_hbm_gbs=byt / attn_us / 1e3,
                   attn_frac_of_hbm_peak=byt / (attn_us * 1e-6) / HBM, pool_bytes_of_users=pages * ps * item,
                   dense_bytes_of_users=B * cap * item, blocks=NB, **info)
        if dense:
            st = m.new_state(B, cap)
            m.extend(st, hist[users, :-1].to(dev), hts[users, :-1].to(dev))

            def dense_one():
                st.lengths.copy_(ulens)
                st.items_bound = cap - 1
                return m.extend(st, ids1, ts1)

            dense_ms = graph_ms(dense_one)
            assert torch.equal(one(), dense_one())                 # same users, same items: the same bits
            row.update(dense_extend_us=dense_ms * 1e3, pool_over_dense=ms / dense_ms,
                       dense_attn_kernel_us=harness.mean_launch_us(harness.profile(dense_one, 20), "hstu_attn_extend_kernel"))
        print(json.dumps(row), flush=True)
        del pool
        torch.cuda.empty_cache()


def bench_rqvae_train(dev):
    """The RQ-VAE training kernels next to the torch code they replace, on the same GPU: rq_sinkhorn (one launch, 100 fp64
    iterations) against the reference's Sinkhorn restated in torch fp64, eager and graph-captured, at the training batch and the
    k-means warm-start batch; the device k-means initialisation against the reference's Lloyd loop restated in torch."""
    import time
    import numpy as np
    from genrec_b200.rqvae import kmeans_init_
    from tests import rqvae_train_oracle as O
    info = harness.card(dev)
    g = torch.Generator().manual_seed(3)
    for B in (1024, 20480):
        x, cb = torch.randn(B, 32, generator=g).to(dev) * 0.3, torch.randn(256, 32, generator=g).to(dev) * 0.3
        dist = O.l2_dist(x, cb)
        ours = harness.timed(lambda: Fn.rq_sinkhorn(dist), 20, 3)[0]
        ours_g = graph_ms(lambda: Fn.rq_sinkhorn(dist), reps=5, iters=4)
        eager = harness.timed(lambda: O.sinkhorn(dist), 5, 2)[0]
        graph = graph_ms(lambda: O.sinkhorn(dist), reps=2, iters=3)
        kern = harness.mean_launch_us(harness.profile(lambda: Fn.rq_sinkhorn(dist), 10), "rq_sinkhorn_kernel")
        print(json.dumps(dict(kernel="rq_sinkhorn", B=B, K=256, iters=100, kernel_us=kern, us=ours * 1e3, graph_us=ours_g * 1e3,
                              torch_fp64_eager_us=eager * 1e3, torch_fp64_graph_us=graph * 1e3, speedup_vs_torch_graph=graph / ours_g,
                              kernel_us_per_iteration=kern / 100, **info)), flush=True)
    x = (torch.randn(256, 32, generator=g)[torch.arange(20480) % 256] + 0.1 * torch.randn(20480, 32, generator=g)).to(dev)
    w = torch.empty(256, 32, device=dev)
    for name, fn in (("ours", lambda: kmeans_init_(w, x)), ("torch_reference_loop", lambda: O.kmeans(x, 256))):
        fn()
        np.random.seed(0)
        torch.manual_seed(0)
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t) * 1e3
        it = r if name == "ours" else r[1]
        print(json.dumps(dict(kernel="kmeans_init", impl=name, B=20480, D=32, k=256, iterations=it, ms=ms, ms_per_iteration=ms / (it + 1),
                              **info)), flush=True)


def bench_linear_bwd(dev):
    """Fn.linear_bwd (dx, dW and db) at the SASRec shapes (configs[0]: B = 128, L = 50, d = 64, FFN 256) and at the T5 projection
    shapes of TIGER (d_model 384, kv projection 768; batch 256, 61 encoder and 4 decoder tokens per sequence), then one SASRec
    training step (forward + backward) at configs[0] geometry.  Graph-captured device time.  Only the Python API is used, so the
    script times any tree that has it."""
    from genrec_b200.sasrec import SASRec
    info = harness.card(dev)
    g = torch.Generator().manual_seed(0)
    shapes = [("sasrec", 6400, 64, 64), ("sasrec", 6400, 256, 64), ("sasrec", 6400, 64, 256),
              ("tiger_encoder", 256 * 61, 384, 384), ("tiger_encoder", 256 * 61, 768, 384),
              ("tiger_decoder", 256 * 4, 384, 384), ("tiger_decoder", 256 * 4, 768, 384)]
    for geo, T, N, K in shapes:
        dy = (torch.randn(T, N, generator=g) * 0.1).to(dev).bfloat16()
        w = (torch.randn(N, K, generator=g) * 0.1).to(dev).bfloat16()
        x = torch.randn(T, K, generator=g).to(dev).bfloat16()
        ms = graph_ms(lambda: Fn.linear_bwd(dy, w, x))
        print(json.dumps(dict(kernel="linear_bwd", geometry=geo, T=T, N=N, K=K, us=ms * 1e3, **info)), flush=True)
    B, L, V = 128, 50, 1000
    torch.manual_seed(0)
    m = SASRec(V, L, 64, 2, 2, 256, dropout=0.2).to(dev).train()
    ids = torch.randint(1, V + 1, (B, L), generator=g)
    ids[torch.arange(L)[None, :] < torch.randint(0, L - 1, (B, 1), generator=g)] = 0      # left padding
    tg = torch.roll(ids, -1, 1)
    ids, tg = ids.to(dev), tg.to(dev)
    for p in m.parameters():
        p.grad = torch.zeros_like(p)

    def step():
        for p in m.parameters():
            p.grad.zero_()
        m(ids, tg)[1].backward()

    ms = graph_ms(step)
    print(json.dumps(dict(kernel="sasrec_train_step", B=B, L=L, D=64, blocks=2, num_items=V, dropout=0.2, ms=ms, **info)), flush=True)


def bench_tiger(dev):
    """TIGER at config/tiger/amazon/tiger.gin shape: one training step (forward, backward, AdamW) at B = 256, and generate at B = 256,
    K = 10 with a 12,000-item trie - eager, replayed from a CUDA graph, and the uncached tiger_decode.generate loop (the reference's
    schedule: memory expanded to every beam) on the same module, the three alternated in rounds."""
    from genrec_b200 import tiger_decode as td
    from genrec_b200.tiger import Tiger
    from tests import tiger_params as tp
    info = harness.card(dev)
    cfg = dict(tp.PUBLISHED, dropout=0.1)
    B, K = 256, 10
    m = Tiger(**cfg)
    m.load_state_dict(tp.tiger_params([(k, v.shape) for k, v in m.state_dict().items()], 3))
    m = m.to(dev)
    b = {k: v.to(dev) for k, v in tp.batch(cfg, B, 20, 5).items()}
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4, weight_decay=0.035, fused=True)

    def step():
        opt.zero_grad(set_to_none=False)
        m(**b).loss.backward()
        opt.step()

    m.train()
    ms = harness.timed(step, 20, 5)[0]
    print(json.dumps(dict(kernel="tiger_train_step", B=B, history_items=20, dropout=0.1, optimizer="AdamW (torch fused)", ms=ms, **info)),
          flush=True)
    m.eval()
    valid = torch.randint(0, 256, (12000, 3), generator=torch.Generator().manual_seed(1))
    m._grb_trie = td.TrieCSR.build(valid).to(dev)
    args = (b["user_input_ids"], b["item_input_ids"], b["token_type_ids"], b["seq_mask"])
    eager = lambda: m.generate(*args, n_top_k_candidates=K)                 # noqa: E731
    uncached = lambda: td.generate(m, *args, n_top_k_candidates=K)          # noqa: E731
    for _ in range(2):
        eager(), uncached()
    graph, _ = harness.graphed(eager, 1)
    rows = {"eager": [], "graph": [], "uncached": []}
    for _ in range(3):
        rows["eager"].append(harness.timed(eager, 10, 1)[0])
        rows["graph"].append(harness.timed(graph.replay, 10, 1)[0])
        rows["uncached"].append(harness.timed(uncached, 10, 1)[0])
    for name, v in rows.items():
        print(json.dumps(dict(kernel="tiger_generate_" + name, B=B, K=K, trie_items=12000, ms_per_round=v, ms=min(v), **info)), flush=True)
    print(json.dumps(dict(kernel="tiger_generate_speedup", eager_vs_uncached=min(rows["uncached"]) / min(rows["eager"]),
                          graph_vs_uncached=min(rows["uncached"]) / min(rows["graph"]))), flush=True)
    del graph
    bench_tiger_wide(dev, m, args, info)


def bench_tiger_wide(dev, m, args, info):
    """Retrieval-sized beams at B = 256 on the published model and a 12,000-item trie: Tiger.generate at K = 64, 256, 1024 (eager and
    replayed from a CUDA graph, alternated in rounds) with its peak memory; per decode step, the device time of the beam-select
    launches next to that step's torch.multinomial (torch.profiler, a run of its own); and the beam step alone at K = 10, where
    both the one-CTA kernel and the wide path apply."""
    from torch.profiler import record_function
    from genrec_b200 import _lib
    from genrec_b200 import tiger_decode as td
    from genrec_b200._lib import ptr, stream_ptr
    B = 256
    for K in (10, 64, 256, 1024):
        gen = lambda: m.generate(*args, n_top_k_candidates=K)                  # noqa: E731
        gen()
        base = torch.cuda.memory_allocated()
        peak = harness.peak(gen) - base
        graph, _ = harness.graphed(gen, 1)
        rows = {"eager": [], "graph": []}
        iters = 10 if K <= 64 else 3
        for _ in range(3):
            rows["eager"].append(harness.timed(gen, iters, 1)[0])
            rows["graph"].append(harness.timed(graph.replay, iters, 1)[0])
        del graph
        torch.cuda.empty_cache()
        if K > 10:
            for name, v in rows.items():
                print(json.dumps(dict(kernel="tiger_generate_" + name, B=B, K=K, trie_items=12000, ms_per_round=v, ms=min(v),
                                      peak_extra_bytes=peak, **info)), flush=True)
        # per-step device time: the beam step's launches (a record_function range around tiger_decode.beam_select) and the
        # step's torch.multinomial, over 3 generate calls of 3 steps each
        orig = td.beam_select

        def traced(*a, **k):
            with record_function("grb_beam_step"):
                return orig(*a, **k)

        td.beam_select = traced
        try:
            prof = harness.profile(gen, 3, 0, cpu=True)
        finally:
            td.beam_select = orig
        steps = 3 * m.sem_id_dim
        ev = {k: us / steps for k, (us, _) in prof.items()}
        kern = {harness.short_name(k): round(v, 1) for k, v in ev.items() if "beam_" in k}
        print(json.dumps(dict(kernel="tiger_beam_step_vs_multinomial", B=B, K=K, KK=min(6 * K, 256), us_beam_step=round(ev.get("grb_beam_step", 0), 1),
                              us_multinomial=round(ev.get("aten::multinomial", 0), 1), kernels_us_per_step=kern,
                              us_trie_log_softmax=round(sum(v for k, v in ev.items() if "trie_log_softmax_kernel" in k), 1), **info)), flush=True)
    # the beam step alone at K = 10 (KK = 60, second step): the one-CTA kernel against the wide path, alternated
    lib = _lib.load()
    g = torch.Generator().manual_seed(4)
    K, KK, S = 10, 60, 1
    valid = torch.randint(0, 256, (12000, 3), generator=g)
    trie = td.TrieCSR.build(valid).to(dev)
    seqs = valid[torch.randint(0, 12000, (B, K), generator=g)][:, :, :S].contiguous().to(dev)
    off, toks, kids = trie.child_off.tolist(), trie.child_tok.tolist(), trie.child_node.tolist()
    root = dict(zip(toks[off[0]:off[1]], kids[off[0]:off[1]]))
    nodes = torch.tensor([[root.get(t, -1) for t in r] for r in seqs[..., 0].tolist()], dtype=torch.int32, device=dev)
    logps = (-torch.rand(B, K, generator=g) * 3).to(dev)
    tok = torch.stack([torch.randperm(256, generator=g)[:KK] for _ in range(B * K)]).view(B, K, KK).to(dev)
    clogp = (-torch.rand(B, K, KK, generator=g) * 5).to(dev)
    out_s, out_l = torch.empty(B, K, S + 1, dtype=torch.long, device=dev), torch.empty(B, K, device=dev)
    out_n = torch.empty(B, K, dtype=torch.int32, device=dev)
    ws = torch.empty(lib.grb_beam_select_wide_workspace_bytes(B, K, KK), dtype=torch.uint8, device=dev)
    a = (ptr(seqs), ptr(logps), ptr(tok), ptr(clogp), ptr(nodes), ptr(trie.child_off), ptr(trie.child_tok), ptr(trie.child_node), trie.n_nodes,
         B, K, KK, S, ptr(out_s), ptr(out_l), ptr(out_n))
    calls = {"one_cta": lambda: lib.grb_beam_select(*a, stream_ptr(dev)), "wide": lambda: lib.grb_beam_select_wide(*a, ptr(ws), stream_ptr(dev))}
    res = {}
    for name, fn in calls.items():
        assert fn() == 0
        torch.cuda.synchronize()
        res[name] = (out_s.clone(), out_l.clone(), out_n.clone())
    same = all(torch.equal(x, y) for x, y in zip(res["one_cta"], res["wide"]))
    rows = {n: [] for n in calls}
    for _ in range(5):
        for n, fn in calls.items():
            rows[n].append(graph_ms(fn) * 1e3)
    for n, v in rows.items():
        print(json.dumps(dict(kernel="tiger_beam_step_k10_" + n, B=B, K=K, KK=KK, S=S, us_per_round=v, us=min(v), same_beams=same, **info)),
              flush=True)


def bench_hstu_attn(dev):
    """Fn.hstu_attention_bwd alone, replayed from a CUDA graph, at the benchmark's two geometries (cfg2: B = 128, L = 200, D = 128,
    H = 4; cfg3: B = 32, L = 2048, D = 256, H = 8), uniform position buckets, with and without the 64-bucket time table.  The call
    also clears its dzp output.  The attention kernels' device time per call comes from a torch.profiler run of its own."""
    from genrec_b200.hstu import _thresholds_on
    info = harness.card(dev)
    for name, B, L, D, H in (("cfg2", 128, 200, 128, 4), ("cfg3", 32, 2048, 256, 8)):
        g = torch.Generator().manual_seed(0)
        zp = (0.7 * torch.randn(B, L, 4 * D, generator=g)).bfloat16().to(dev)
        P = torch.nn.functional.silu(zp.float()).bfloat16()
        dO = (torch.randn(B, L, D, generator=g) / L ** 0.5).bfloat16().to(dev)
        ts = (1_300_000_000 + torch.cumsum(torch.randint(1, 3 * 86400, (B, L), generator=g), 1)).to(dev)
        pad = torch.zeros(B, L, dtype=torch.uint8, device=dev)
        pb = torch.zeros(L, dtype=torch.uint8, device=dev)
        wpos, wtime = (0.3 * torch.randn(32, H, generator=g)).to(dev), (0.5 * torch.randn(64, H, generator=g)).to(dev)
        for time_table in (True, False):
            meta = Fn.SeqMeta(pad, ts if time_table else None, pb, _thresholds_on(dev), 64, 32, (True, 0))
            wt = wtime if time_table else None

            def call():
                return Fn.hstu_attention_bwd(P, zp, dO, meta, H, wpos, wt, 64)

            ms = graph_ms(call)
            iters = 20
            kern = {harness.short_name(k, "<"): round(us / iters, 2) for k, (us, _) in harness.profile(call, iters).items()
                    if "hstu_attn_bwd" in k or "det_finish" in k}
            print(json.dumps(dict(kernel="hstu_attention_bwd", geometry=name, B=B, L=L, D=D, H=H, time_table=time_table,
                                  us=ms * 1e3, kernel_us_per_call=kern, **info)), flush=True)


def main():
    dev = torch.device("cuda:0")
    if sys.argv[1:] == ["hstu_attn"]:
        bench_hstu_attn(dev)
        return
    if sys.argv[1:] == ["rqvae_train"]:
        bench_rqvae_train(dev)
        return
    if sys.argv[1:] == ["linear_bwd"]:
        bench_linear_bwd(dev)
        return
    if sys.argv[1:] == ["head_topk"]:
        bench_head_topk(dev)
        return
    if sys.argv[1:] == ["tiger"]:
        bench_tiger(dev)
        return
    if sys.argv[1:] == ["head_rank"]:
        bench_head_rank(dev)
        return
    if sys.argv[1:] == ["head_candidates"]:
        bench_head_candidates(dev)
        return
    peaks = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json"))) \
        if os.path.exists("MEASURED_PEAKS.json") else {}
    g = torch.Generator().manual_seed(0)
    # ---- RQ-VAE residual argmin (cfg-4): 3 levels x 256 codes, latent 32
    cbs = torch.stack([(torch.rand(256, 32, generator=g) - 0.5) / 2 ** l for l in range(3)]).to(dev)
    for N in (12101, 1 << 20):
        x = torch.randn(N, 32, generator=g).to(dev)
        for aux in (False, True):
            for mode in ("auto", "tile", "split", "thread"):
                if mode == "auto":
                    os.environ.pop("GRB_RQ", None)
                else:
                    os.environ["GRB_RQ"] = mode
                ms = graph_ms(lambda: Fn.rq_residual_argmin(x, cbs, 0.25, want_aux=aux))
                flops = 2 * 256 * 32 * 3 * N
                byt = N * (32 * 4 + 3 * 8 + (2 * 32 * 3 * 4 + 4 if aux else 0))
                print(json.dumps(dict(kernel="rq_residual_argmin", N=N, aux_outputs=aux, dispatch=mode, us=ms * 1e3, items_per_s=N / ms * 1e3,
                                      fp32_tflops=flops / ms / 1e9, hbm_gbs=byt / ms / 1e6,
                                      note="graph-captured device time; FP32 FMA bound by specification (no tensor cores)")))
            os.environ.pop("GRB_RQ", None)
    # ---- HSTU layer fwd+bwd at cfg-3 geometry
    for (B, L, D, H) in ((16, 2048, 256, 8), (128, 200, 128, 4)):
        layer = HSTULayer(D, H, 0.0, 32, 64, 128, True).to(dev).train()
        ts = (1_300_000_000 + torch.cumsum(torch.randint(1, 3 * 86400, (B, L), generator=g), 1)).to(dev)
        pad = torch.zeros(B, L, dtype=torch.bool, device=dev)
        x = torch.randn(B, L, D, generator=g).to(dev).requires_grad_(True)
        dy = torch.randn(B, L, D, generator=g).to(dev)

        def fb():
            y = layer(x, None, pad, ts)
            y.backward(dy)

        ms = harness.timed(fb, 10, 3)[0]
        flops = (72 * L * D * D + 6 * D * L * (L + 1)) * B
        peak = peaks.get("bf16_tflops", 989.0)   # H100 SXM data sheet, dense bf16 at 700 W
        print(json.dumps(dict(kernel="hstu_layer_fwd_bwd", B=B, L=L, D=D, H=H, ms=ms, seq_per_s=B / ms * 1e3,
                              algorithmic_tflops=flops / ms / 1e9, frac_of_bf16_peak=flops / ms / 1e9 / peak,
                              note="eager launches (not graph-captured): includes host launch gaps at L=200")))
    bench_extend(dev)
    bench_pool(dev)
    bench_rqvae_train(dev)


if __name__ == "__main__":
    main()
