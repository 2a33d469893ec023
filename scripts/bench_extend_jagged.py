"""Serving calls of HSTU on packed (jagged) chunks against the padded chunks of the same items: extend_users_jagged against
extend_users on a paged pool.

Geometries: cfg2 (V = 12,101 items, D = 128, 4 heads, 4 blocks) and cfg3 (D = 256, 8 heads, 8 blocks).  Each workload draws one
seeded call: B users of the pool and each user's new items.  The padded call takes them as a left-padded [B, n] chunk with n the
longest; the packed call takes them as T = the sum of the lengths token rows.  Both calls use device users and device offsets,
are captured in a CUDA graph after one eager call and replayed; every replay first restores the pool's bookkeeping (lengths,
overflow flags, page table, free stack) to the snapshot taken before the call, so that each replay does the same work.  The two
graphs are timed with CUDA events, alternated three times in one process (medians).  The two paths' first-call logits must be
torch.equal before anything is timed.  ``--profile`` adds a torch.profiler per-kernel breakdown of one eager call of each path.

    python scripts/bench_extend_jagged.py [--steps 20] [--workloads cfg2_prefill,...] [--profile cfg2_prefill]

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

CFG2 = dict(num_items=12101, embed_dim=128, num_heads=4, num_blocks=4)
CFG3 = dict(num_items=12101, embed_dim=256, num_heads=8, num_blocks=8)
WORKLOADS = {   # name: (geometry, pool users, max_items, B, history before the call, new items per user, description, aim)
    "cfg2_prefill": (CFG2, 4096, 200, 128, None, ("uniform", 1, 199), "cfg2 pool prefill, lengths U[1, 199]", "<= 0.65"),
    "cfg3_prefill": (CFG3, 512, 2048, 32, None, ("uniform", 1, 2047), "cfg3 pool prefill, lengths U[1, 2047]", "<= 0.65"),
    "cfg2_events": (CFG2, 4096, 200, 128, ("uniform", 1, 150), ("geometric", 1, 16),
                    "cfg2 pool, each user adds geometric 1..16 new items (mean about 4)", "none"),
    "cfg2_equal_1": (CFG2, 4096, 200, 128, ("uniform", 1, 150), ("full", 1, 1), "cfg2 pool, every user adds 1 item", "within 3%"),
    "cfg2_equal_199": (CFG2, 4096, 200, 128, None, ("full", 199, 199), "cfg2 pool, full 199-item prefills", "within 3%"),
}


def user_lengths(rule, B, g):
    """B users' item counts under a workload's (kind, lo, hi) rule; geometric has mean 4, cut at hi"""
    kind, lo, hi = rule
    if kind == "full":
        return torch.full((B,), hi, dtype=torch.int64)
    if kind == "uniform":
        return torch.randint(lo, hi + 1, (B,), generator=g)
    return harness.geometric_lengths(B, 4, lo, hi, g)


def items_of(lens, V, g, t0):
    """each user's items (power-law ids) and increasing timestamps from t0 [B]"""
    w = torch.arange(1, V + 1, dtype=torch.float64).pow(-1.1)
    ids = [torch.multinomial(w, int(n), replacement=True, generator=g) + 1 for n in lens]
    ts = [int(t) + torch.cumsum(torch.randint(1, 3 * 86400, (int(n),), generator=g), 0) for n, t in zip(lens, t0)]
    return ids, ts


def packed(ids, ts, dev):
    off = torch.zeros(len(ids) + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(torch.tensor([len(i) for i in ids], dtype=torch.int64), 0)
    return torch.cat(ids).to(dev), torch.cat(ts).to(dev), off.to(dev)


def padded(ids, ts, dev):
    n = max(len(i) for i in ids)
    pi = torch.zeros(len(ids), n, dtype=torch.int64)
    pt = torch.zeros(len(ids), n, dtype=torch.int64)
    for b, (i, t) in enumerate(zip(ids, ts)):
        pi[b, n - len(i):] = i
        pt[b, n - len(i):] = t
    return pi.to(dev), pt.to(dev)


def setup(name, dev):
    """-> the model, the pool, and the call's users / chunks (padded and packed) with their shapes"""
    from genrec_b200.hstu import HSTU
    geo, nusers, cap, B, hist_rule, new_rule, _, _ = WORKLOADS[name]
    g = torch.Generator().manual_seed(7)
    torch.manual_seed(0)
    m = HSTU(max_seq_len=cap, dropout=0.0, **geo).to(dev).eval()
    users = torch.randperm(nusers, generator=g)[:B]
    t0 = torch.full((B,), 1_300_000_000, dtype=torch.int64)
    hist = user_lengths(hist_rule, B, g) if hist_rule else torch.zeros(B, dtype=torch.int64)
    new = user_lengths(new_rule, B, g)
    pages = int(((hist + new + 63) // 64).sum()) + 8
    pool = m.new_pool(max_users=nusers, num_pages=pages, page_size=64, max_items=cap)
    if hist_rule:
        hids, hts = items_of(hist, geo["num_items"], g, t0)
        ids, ts, off = packed(hids, hts, dev)
        m.extend_users_jagged(pool, users.to(dev), ids, off, int(hist.max()), ts)
        t0 = torch.stack([t[-1] for t in hts])
    nids, nts = items_of(new, geo["num_items"], g, t0)
    return m, pool, users.to(dev), padded(nids, nts, dev), packed(nids, nts, dev), int(new.max())


def run(name, steps, dev, info, profile):
    geo, nusers, cap, B, _, _, desc, aim = WORKLOADS[name]
    m, pool, users, (pi, pt), (ids, ts, off), max_len = setup(name, dev)
    book = [pool.lengths, pool.overflow, pool.page_table, pool.free_stack, pool.free_top, pool.last_hidden]
    snap = [t.clone() for t in book]

    def restore():
        for t, s in zip(book, snap):
            t.copy_(s)

    calls = {"padded": lambda: m.extend_users(pool, users, pi, pt),
             "packed": lambda: m.extend_users_jagged(pool, users, ids, off, max_len, ts)}
    res = {}
    for path, call in calls.items():
        restore()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()           # peak_extra_mb: the call's working memory above what is resident
        torch.cuda.reset_peak_memory_stats()
        first = call()
        torch.cuda.synchronize()
        res[path] = dict(first=first.clone(), peak_mb=(torch.cuda.max_memory_allocated() - base) / 2 ** 20)
        del first
    assert torch.equal(res["padded"]["first"], res["packed"]["first"]), "the packed call's logits differ from the padded call's"
    for path, call in calls.items():
        res[path]["graph"] = harness.graphed(lambda call=call: (restore(), call())[1], 2)[0]
    times = {"padded": [], "packed": []}
    for _ in range(3):
        for path in ("padded", "packed"):
            times[path].append(harness.timed(res[path]["graph"].replay, steps, 1)[0])
    out = dict(workload=name, desc=desc, B=B, pool_users=nusers, max_items=cap, aim=aim, padded_tokens=pi.numel(),
               packed_tokens=ids.numel(), padding_share=round(1 - ids.numel() / pi.numel(), 4), first_call_equal=True, **info)
    for path in ("padded", "packed"):
        out[path] = dict(call_ms=round(statistics.median(times[path]), 4), runs_ms=[round(t, 4) for t in times[path]],
                         peak_extra_mb=round(res[path]["peak_mb"], 1))
    out["packed_over_padded"] = round(out["packed"]["call_ms"] / out["padded"]["call_ms"], 4)
    if profile:
        for path, call in calls.items():
            res[path]["graph"].reset()
            kernels = harness.largest_first(harness.profile(lambda call=call: (restore(), call())[1]), lambda k: harness.short_name(k)[:60])
            out[path]["kernels_us"] = {k: round(us, 1) for k, us in kernels.items()}
    print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--profile", default="cfg2_prefill", help="workloads that also get a per-kernel torch.profiler breakdown")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_extend_jagged.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    info = harness.card(dev)
    prof = set(args.profile.split(",")) if args.profile else set()
    for name in args.workloads.split(","):
        run(name, args.steps, dev, info, name in prof)


if __name__ == "__main__":
    main()
