"""Generate tests/golden/tiger_small_dropout*.pt from the UNMODIFIED reference Tiger (needs the reference tree, see oracle/ref_loader.py).

    python scripts/make_golden_tiger_dropout.py

One training step of tiger_small.pt's model (tests/tiger_params.SMALL, the same parameter seed and batch) at dropout 0.3, in fp64.
Every nn.Dropout module of the reference (Tiger.drop, each T5Attention's dropout on the probabilities, dropout1, dropout_cross, the
FFN's hidden dropout, dropout2) is replaced by one that multiplies its input by the next of a list of pre-drawn keep-scale masks, in
call order, at the kernels' keep scale (tests/attention_reference.keep_scale).  The reference's norms cast to fp32 for the mean of
squares (normalize.py:54, :89); a torch function mode keeps those casts of fp64 tensors in fp64, so the whole step is fp64.

The fixture stores the masks (bool keep [shape], in call order), logits, loss and every parameter gradient; the four FFN weight
gradients go in one part each (tests/conftest.py merges <stem>.<key>.pt parts) so every file stays under 1 MB.
"""
from __future__ import annotations

import os
import sys

import torch
from torch.overrides import TorchFunctionMode

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from tests import tiger_params as tp  # noqa: E402
from tests.attention_reference import keep_scale  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
P, PARAM_SEED, BATCH_SEED, MASK_SEED, B, N_ITEMS = 0.3, 1, 2, 11, 4, 5


class _KeepFp64(TorchFunctionMode):
    """x.float() / x.to(torch.float32) of an fp64 tensor returns it unchanged"""

    def __torch_function__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        x = args[0] if args else None
        if isinstance(x, torch.Tensor) and x.dtype == torch.float64:
            if func is torch.Tensor.float or (func is torch.Tensor.to and torch.float32 in tuple(args[1:]) + tuple(kwargs.values())):
                return x
        return func(*args, **kwargs)


def _run(m, batch, masks):
    """one forward + backward with every nn.Dropout replaced: masks None records the shapes, else applies them in order"""
    shapes, it = [], iter(masks or [])

    def drop(x):
        if masks is None:
            shapes.append(tuple(x.shape))
            return x
        k = next(it)
        assert tuple(k.shape) == tuple(x.shape)
        return x * k.to(x.dtype)

    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.forward = drop
    m.zero_grad(set_to_none=True)
    with _KeepFp64():
        out = m(**batch)
        out.loss.backward()
    assert next(it, None) is None
    return out, shapes


def main():
    assert ref_loader.available(), "reference tree not found"
    tg = ref_loader.ref_tiger()
    cfg = dict(tp.SMALL, dropout=P)
    m = tg.Tiger(**cfg)
    shapes = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    m.load_state_dict(tp.tiger_params(shapes, PARAM_SEED), strict=True)
    m = m.double().train()
    batch = tp.batch(cfg, B, N_ITEMS, BATCH_SEED)
    _, mshapes = _run(m, batch, None)
    g = torch.Generator().manual_seed(MASK_SEED)
    keep = [torch.rand(s, generator=g, dtype=torch.float64) >= P for s in mshapes]
    scale = keep_scale(P)[1]
    out, _ = _run(m, batch, [k.double() * scale for k in keep])
    grads = {n: p.grad.clone() for n, p in m.named_parameters() if p.grad is not None}
    big = {n for n, t in grads.items() if t.numel() >= 65536}
    torch.save(dict(cfg=cfg, param_seed=PARAM_SEED, batch_seed=BATCH_SEED, B=B, n_items=N_ITEMS, shapes=shapes, p=P, keep=keep,
                    logits=out.logits.detach().clone(), loss=out.loss.detach().clone(),
                    grads={n: t for n, t in grads.items() if n not in big}), os.path.join(OUT, "tiger_small_dropout.pt"))
    for n in sorted(big):
        torch.save({n: grads[n]}, os.path.join(OUT, "tiger_small_dropout.grads_" + n.replace(".", "_") + ".pt"))
    for f in sorted(os.listdir(OUT)):
        if f.startswith("tiger_small_dropout"):
            print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()
