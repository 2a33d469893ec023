"""Stand-alone device timings of the secondary kernels (RQ-VAE residual argmin, SASRec attention, HSTU layer at cfg-3 geometry,
cached incremental HSTU inference next to full recompute) with CUDA events, against the relevant roofline.  Prints one JSON line per
measurement."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import genrec_b200.functional as Fn
from genrec_b200.hstu import HSTULayer


def timed(fn, iters=20, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def graph_timed(fn, reps=10, iters=10):
    """Device time per call with the launches captured in a CUDA graph (no host gaps: what a small kernel really costs)."""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(reps):
                fn()
        g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (reps * iters)


def kernel_us(fn, name, iters=20):
    """Mean device time (us) per launch of the kernels whose name contains `name`, from a torch.profiler run of its own."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    hits = [k for k in prof.key_averages() if name in k.key]
    total, count = sum(k.device_time_total for k in hits), sum(k.count for k in hits)
    return total / count if count else float("nan")


def card():
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True,
                       text=True)
    return dict(gpu=torch.cuda.get_device_name(0), power_limit_and_max_sm_clock=q.stdout.strip() or "unknown")


def bench_extend(dev):
    """Cached incremental inference (HSTU.extend) next to full recompute (HSTU.last_logits) on the same full sequences: one new
    item per user on a history of L - 1, and the prefill of the whole history (extend on an empty state).  Both graph-captured.
    The state is rewound on the device before every call (lengths.fill_, one small kernel inside the timed graph), so every call
    appends at the same position.  The chunk-attention kernel's bytes are the cache K | V and timestamps it must read."""
    from genrec_b200.hstu import HSTU
    info = card()
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

            full_ms = graph_timed(lambda: m.last_logits(ids, ts))
            for work, fn, keys in (("extend_1", one, L), ("prefill", prefill, None)):
                ms = graph_timed(fn)
                row = dict(kernel="hstu_extend", geometry=name, workload=work, B=B, history=L - 1 if work == "extend_1" else 0,
                           new_items=1 if work == "extend_1" else L, extend_us=ms * 1e3, last_logits_us=full_ms * 1e3,
                           speedup_vs_last_logits=full_ms / ms, **info)
                if keys is not None:
                    attn_us = kernel_us(fn, "hstu_attn_extend_kernel")
                    byt = B * keys * (2 * D * 2 + 8)            # per layer: K | V bf16 + int64 timestamp of every cached key
                    row.update(attn_kernel_us=attn_us, attn_bytes_per_layer=byt, attn_hbm_gbs=byt / attn_us / 1e3,
                               attn_frac_of_hbm_peak=byt / (attn_us * 1e-6) / HBM, blocks=NB)
                print(json.dumps(row), flush=True)
            assert torch.isfinite(one()).all()


def bench_pool(dev):
    """Serving from the paged pool (HSTU.extend_users): a pool of many users with seeded history lengths, one new item for a random
    subset of them, next to the dense HSTUState extend of the same users (cfg2) and last_logits on their left-padded histories.
    Graph-captured with the users as a device tensor.  Every length is a non-multiple of the page size, so the timed item never
    takes a page, and the lengths are rewound on the device before every call (one small kernel inside the timed graph).  The
    allocation kernel and the chunk-attention kernel are timed on their own with torch.profiler."""
    from genrec_b200.hstu import HSTU
    info = card()
    HBM = 3.35e12
    geoms = (("cfg2", dict(num_items=12101, embed_dim=128, num_heads=4, num_blocks=4), 4096, 200, 128, True),
             ("cfg3", dict(num_items=12101, embed_dim=256, num_heads=8, num_blocks=8), 512, 2048, 32, False))
    for name, geo, nusers, cap, B, dense in geoms:
        g = torch.Generator().manual_seed(1)
        torch.manual_seed(0)
        m = HSTU(max_seq_len=cap, dropout=0.0, **geo).to(dev).eval()
        D, NB, ps = geo["embed_dim"], geo["num_blocks"], 64
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

        def one():
            pool.lengths.index_copy_(0, users_dev, ulens)
            return m.extend_users(pool, users_dev, ids1, ts1)

        ms = graph_timed(one)
        hist_u, hts_u = hist[users].to(dev), hts[users].to(dev)
        full_ms = graph_timed(lambda: m.last_logits(hist_u, hts_u))
        attn_us = kernel_us(one, "hstu_attn_extend_kernel")
        alloc_us = kernel_us(one, "hstu_pool_alloc_kernel")
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

            dense_ms = graph_timed(dense_one)
            assert torch.equal(one(), dense_one())                 # same users, same items: the same bits
            row.update(dense_extend_us=dense_ms * 1e3, pool_over_dense=ms / dense_ms,
                       dense_attn_kernel_us=kernel_us(dense_one, "hstu_attn_extend_kernel"))
        print(json.dumps(row), flush=True)
        del pool
        torch.cuda.empty_cache()


def main():
    dev = torch.device("cuda:0")
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
                ms = graph_timed(lambda: Fn.rq_residual_argmin(x, cbs, 0.25, want_aux=aux))
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

        ms = timed(fb, iters=10, warm=3)
        flops = (72 * L * D * D + 6 * D * L * (L + 1)) * B
        peak = peaks.get("bf16_tflops", 989.0)   # H100 SXM data sheet, dense bf16 at 700 W
        print(json.dumps(dict(kernel="hstu_layer_fwd_bwd", B=B, L=L, D=D, H=H, ms=ms, seq_per_s=B / ms * 1e3,
                              algorithmic_tflops=flops / ms / 1e9, frac_of_bf16_peak=flops / ms / 1e9 / peak,
                              note="eager launches (not graph-captured): includes host launch gaps at L=200")))
    bench_extend(dev)
    bench_pool(dev)


if __name__ == "__main__":
    main()
