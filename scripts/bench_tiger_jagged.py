"""TIGER training step and beam search on a packed (jagged) encoder memory against pad_collate's padded batch of the same users.

Published shape (config/tiger/amazon/tiger.gin): embedding 128, attention 384, 6 heads, 8 layers, 256 codes x 3, max_seq_len 20 items
(61 memory tokens with the user token).  For each workload one seeded set of users is drawn (item counts geometric with mean 9,
capped at 20, or all 20); the padded path runs Tiger.forward / generate on the batch padded to its longest history, the packed path
forward_jagged / generate_jagged on data.pack_tiger of it.  Dropout is 0, so the first-step losses must be equal.

- Training step: forward, backward and torch's fused AdamW, eager (the step is not captured), timed with CUDA events.
- generate: captured in a CUDA graph and replayed, timed with CUDA events.
Each pair is alternated three times in one process; medians.  Peak memory is torch.cuda.max_memory_allocated over one step (one eager call for generate).
``--profile`` writes a torch.profiler per-kernel split of one training step of each path into ``--out`` (by default a new temporary
directory, so nothing is written into the source tree; its path is printed).

    python scripts/bench_tiger_jagged.py [--steps 20] [--out DIR] [--profile] [--workloads train_geo1024,...]

Prints one JSON line per workload."""
import argparse
import json
import os
import statistics
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from scripts import harness  # noqa: E402

CFG = dict(embedding_dim=128, attn_dim=384, dropout=0.0, num_heads=6, n_layers=8, num_item_embeddings=256, num_user_embeddings=10000,
           sem_id_dim=3)
MAX_ITEMS = 20
WORKLOADS = {   # name: (kind, B, lengths, aim on packed / padded)
    "train_geo256": ("train", 256, "geometric", "none (bound by launches)"),
    "train_geo1024": ("train", 1024, "geometric", "<= 0.7"),
    "train_full256": ("train", 256, "full", "within 3%"),
    "train_full1024": ("train", 1024, "full", "within 3%"),
    "gen10_geo": ("generate10", 256, "geometric", "none"),
    "gen256_geo": ("generate256", 256, "geometric", "<= 0.8"),
    "gen10_full": ("generate10", 256, "full", "within 3%"),
    "gen256_full": ("generate256", 256, "full", "within 3%"),
}


def batch(B, kind, seed, dev):
    """-> (padded dict as pad_collate makes it, packed dict of data.pack_tiger), both on dev"""
    from genrec_b200.data import pack_tiger
    rng = np.random.default_rng(seed)
    n = np.full(B, MAX_ITEMS) if kind == "full" else np.minimum(rng.geometric(1.0 / 9, B), MAX_ITEMS)
    C, E = CFG["sem_id_dim"], CFG["num_item_embeddings"]
    W = int(n.max()) * C
    toks = [torch.from_numpy(rng.integers(0, E, int(k) * C)) for k in n]
    users = torch.from_numpy(rng.integers(0, 10 ** 6, B))
    target = torch.from_numpy(rng.integers(0, E, (B, C)))
    ids = torch.zeros(B, W, dtype=torch.int64)
    types = torch.zeros(B, W, dtype=torch.int64)
    mask = torch.zeros(B, W, dtype=torch.int64)
    for b, t in enumerate(toks):
        ids[b, :len(t)] = t
        types[b, :len(t)] = torch.arange(len(t)) % 3
        mask[b, :len(t)] = 1
    padded = dict(user_input_ids=users.view(B, 1), item_input_ids=ids, token_type_ids=types, target_input_ids=target,
                  target_token_type_ids=torch.arange(C).expand(B, C).contiguous(), seq_mask=mask)
    padded = {k: v.to(dev) for k, v in padded.items()}
    off = torch.zeros(B + 1, dtype=torch.int64)
    off[1:] = torch.from_numpy(np.cumsum(n * C))
    packed = pack_tiger(users.to(dev), torch.cat(toks).to(dev), off.to(dev), target.to(dev), max_items=MAX_ITEMS)
    return padded, packed


def model(dev):
    from genrec_b200.tiger import Tiger
    from tests import tiger_params as tp
    m = Tiger(**CFG)
    m.load_state_dict(tp.tiger_params([(k, v.shape) for k, v in m.state_dict().items()], 7))
    return m.to(dev)


def train_fns(m, padded, packed):
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4, weight_decay=0.035, fused=True)

    def step_padded():
        opt.zero_grad(set_to_none=True)
        out = m(padded["user_input_ids"], padded["item_input_ids"], padded["token_type_ids"], padded["target_input_ids"],
                padded["target_token_type_ids"], padded["seq_mask"])
        out.loss.backward()
        opt.step()
        return out.loss

    def step_packed():
        opt.zero_grad(set_to_none=True)
        out = m.forward_jagged(packed["user_input_ids"], packed["item_input_ids"], packed["token_type_ids"], packed["mem_offsets"],
                               packed["max_len"], packed["target_input_ids"], packed["target_token_type_ids"])
        out.loss.backward()
        opt.step()
        return out.loss
    return step_padded, step_packed


def gen_fns(m, padded, packed, K, valid):
    def padded_call():
        return m.generate(padded["user_input_ids"], padded["item_input_ids"], padded["token_type_ids"], padded["seq_mask"],
                          n_top_k_candidates=K, valid_item_ids=valid)

    def packed_call():
        return m.generate_jagged(packed["user_input_ids"], packed["item_input_ids"], packed["token_type_ids"], packed["mem_offsets"],
                                 packed["max_len"], n_top_k_candidates=K, valid_item_ids=valid)
    return [padded_call, packed_call]


def peak_mb(fn):
    """MiB allocated at the peak of one call of fn, above what was allocated before it"""
    base = torch.cuda.memory_allocated()
    return (harness.peak(fn) - base) / 2 ** 20


def profile_to(fn, path):
    """one call of fn under torch.profiler, after one untimed call: writes each kernel's device us to `path`, largest first, and
    returns their sum in ms"""
    kernels = harness.largest_first(harness.profile(fn))
    with open(path, "w") as f:
        for k, v in kernels.items():
            f.write(f"{v:10.1f} us  {k}\n")
    return sum(kernels.values()) / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--out", default=None, help="directory for the --profile files (default: a new temporary directory)")
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    if a.profile and a.out is None:
        a.out = tempfile.mkdtemp(prefix="bench_tiger_jagged_")
        print(f"profiles: {a.out}", flush=True)
    dev = torch.device("cuda:0")
    info = harness.card(dev)
    valid = torch.randint(0, CFG["num_item_embeddings"], (20000, 3), generator=torch.Generator().manual_seed(2))
    for name in a.workloads.split(","):
        kind, B, lengths, aim = WORKLOADS[name]
        padded, packed = batch(B, lengths, 11, dev)
        m = model(dev)
        res = dict(workload=name, B=B, lengths=lengths, aim=aim, **info,
                   tokens_padded=int(padded["seq_mask"].numel() + B), tokens_packed=int(packed["item_input_ids"].numel()))
        if kind == "train":
            m.train()
            with torch.no_grad():                                                # the same weights, before any update
                res["loss_padded"] = float(m(padded["user_input_ids"], padded["item_input_ids"], padded["token_type_ids"],
                                             padded["target_input_ids"], padded["target_token_type_ids"], padded["seq_mask"]).loss)
                res["loss_packed"] = float(m.forward_jagged(packed["user_input_ids"], packed["item_input_ids"], packed["token_type_ids"],
                                                            packed["mem_offsets"], packed["max_len"], packed["target_input_ids"],
                                                            packed["target_token_type_ids"]).loss)
            fns = train_fns(m, padded, packed)
            res["peak_mb"] = [round(peak_mb(f), 1) for f in fns]
            if a.profile:
                os.makedirs(a.out, exist_ok=True)
                res["profiled_ms"] = [round(profile_to(f, os.path.join(a.out, f"prof_{name}_{p}.txt")), 3)
                                      for f, p in zip(fns, ("padded", "packed"))]
        else:
            m.eval()
            eager = gen_fns(m, padded, packed, 10 if kind == "generate10" else 256, valid)
            res["peak_mb"] = [round(peak_mb(f), 1) for f in eager]       # one eager call: a replay allocates nothing
            fns = [harness.graphed(f, 2)[0].replay for f in eager]
        for f in fns:
            for _ in range(3):
                f()
        t = {0: [], 1: []}
        for _ in range(3):
            for i, f in enumerate(fns):
                t[i].append(harness.timed(f, a.steps, 0)[0])
        res["ms_padded"], res["ms_packed"] = statistics.median(t[0]), statistics.median(t[1])
        res["ratio"] = round(res["ms_packed"] / res["ms_padded"], 3)
        res["runs_ms"] = {"padded": [round(x, 3) for x in t[0]], "packed": [round(x, 3) for x in t[1]]}
        print(json.dumps(res), flush=True)
        del m, fns
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
