"""Stand-alone device timings of the secondary kernels (RQ-VAE residual argmin, SASRec attention, HSTU layer at cfg-3
geometry) with CUDA events, against the relevant roofline.  Prints one JSON line per measurement."""
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


if __name__ == "__main__":
    main()
