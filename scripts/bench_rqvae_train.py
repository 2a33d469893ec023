"""One RQ-VAE training step at TIGER geometry (768 -> 512 -> 256 -> 128 -> 64 -> 32, 3 x 256 codes, STE / STE / SINKHORN), B = 1024:
forward, backward, clip_grad_norm_(1.0) and AdamW, as genrec/trainers/rqvae_trainer.py runs it.  genrec_b200.rqvae.RqVae against the
same model restated in plain torch (tests/rqvae_train_oracle.py: the reference's 100-iteration fp64 Sinkhorn loop), each eager and
captured in a CUDA graph.  Prints one JSON line per variant."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from genrec_b200.rqvae import QuantizeForwardMode as M, RqVae
from scripts.bench_kernels import card
from tests import rqvae_train_oracle as O

GEO = dict(input_dim=768, hidden=[512, 256, 128, 64], D=32, levels=3, K=256)
MODES = ["STE", "STE", "SINKHORN"]


def step_fn(kind, dev):
    state = O.seeded_state(GEO["input_dim"], GEO["hidden"], GEO["D"], GEO["levels"], GEO["K"], seed=1)
    if kind == "ours":
        m = RqVae(input_dim=768, embed_dim=32, hidden_dims=GEO["hidden"], codebook_size=256, codebook_kmeans_init=False,
                  codebook_mode=M.STE, codebook_last_layer_mode=M.SINKHORN, n_layers=3, n_cat_features=0)
        m.load_state_dict(state)
        m = m.to(dev).train()
        params = list(m.parameters())
        loss_fn = lambda b: m(b, 0.2).loss                                             # noqa: E731
    else:
        p = {k: v.to(dev).requires_grad_(True) for k, v in state.items()}
        params = list(p.values())
        loss_fn = lambda b: O.train_forward(p, b, MODES)[0]["loss"]                    # noqa: E731
    opt = torch.optim.AdamW(params, lr=1e-3, weight_decay=1e-4, capturable=True)
    batch = O.seeded_items(1024, 768, seed=2).to(dev)

    def step():
        opt.zero_grad(set_to_none=False)
        loss_fn(batch).backward()
        torch.nn.utils.clip_grad_norm_(params, 1.0, foreach=True)
        opt.step()
    return step


def time_eager(fn, iters=30, warm=5):
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


def time_graph(fn, iters=30):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    dev = torch.device("cuda:0")
    info = card()
    for kind in ("ours", "torch_restatement"):
        for mode, timer in (("eager", time_eager), ("cuda_graph", time_graph)):
            ms = timer(step_fn(kind, dev))
            print(json.dumps(dict(bench="rqvae_train_step", impl=kind, mode=mode, B=1024, geometry="tiger", ms=ms, **info)), flush=True)


if __name__ == "__main__":
    main()
