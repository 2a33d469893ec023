"""Generate tests/golden/cobra_small_dropout.pt from the UNMODIFIED reference Cobra (needs the reference tree, see oracle/ref_loader.py).

    python scripts/make_golden_cobra_dropout.py

One training step of cobra_small.pt's model and ragged batch (tests/cobra_params.SMALL, the same seeds) with every dropout at
p = 0.3, the item-text encoder's included, in fp64 on the CPU.  Every dropout draws nothing: each nn.Dropout module multiplies its
input by the next of a list of pre-drawn keep-scale masks, and so does the attention.  nn.MultiheadAttention in training with
need_weights=False hands its probability dropout to scaled_dot_product_attention(..., dropout_p); a torch function mode replaces that
call by the explicit softmax(q k^T scale + mask) keep v (a query row without a key gives 0 and a zero gradient, as torch's math kernel does; the
decoder's cross-attention over the empty memory has no probabilities and takes no mask).  The masks are applied in call order, at
the kernels' keep scale (tests/attention_reference.keep_scale).  Running the script again gives the same bytes.

The masks are drawn from MASK_SEED (keep = torch.rand(shape) >= p, in call order); the fixture stores their shapes and the seed
(tests/cobra_reference.fixture_masks rebuilds them), every CobraOutput field, every vector gradient and SAMPLES seeded entries of every matrix gradient.
"""
from __future__ import annotations

import io
import math
import os
import sys

import torch
import torch.nn.functional as F
from torch.overrides import TorchFunctionMode

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tests import cobra_params as cp  # noqa: E402
from tests import cobra_ref  # noqa: E402
from tests.cobra_reference import fixture_masks  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "cobra_small_dropout.pt")
P, MASK_SEED = 0.3, 13
PARAM_SEED = BATCH_SEED = 109        # cobra_small.pt's seeds (scripts/make_golden_cobra.py)
SAMPLES = 256


class _Masks(TorchFunctionMode):
    """multi_head_attention_forward with its scaled_dot_product_attention (the module global it calls when need_weights=False)
    replaced by explicit math that applies the next mask to the probabilities; every other call unchanged"""

    def __init__(self, take):
        super().__init__()
        self.take = take

    def _sdpa(self, q, k, v, attn_mask=None, dropout_p=0.0, is_causal=False, scale=None):
        if k.shape[-2] == 0:                                  # the empty memory: zeros that still reach q, k, v in the graph
            return (q @ k.transpose(-1, -2)) @ v
        s = (q @ k.transpose(-1, -2)) * (scale or 1.0 / math.sqrt(q.shape[-1]))
        if attn_mask is not None:
            s = s.masked_fill(~attn_mask, float("-inf")) if attn_mask.dtype == torch.bool else s + attn_mask
        if is_causal:
            L, S = s.shape[-2:]
            s = s.masked_fill(torch.ones(L, S, dtype=torch.bool).triu(1), float("-inf"))
        live = torch.isfinite(s).any(-1, keepdim=True)      # a query row without a key: 0, and no NaN in the backward
        p = torch.softmax(torch.where(live, s, torch.zeros_like(s)), -1) * live
        return (self.take(p) if dropout_p > 0 else p) @ v

    def __torch_function__(self, func, types, args=(), kwargs=None):
        kwargs = kwargs or {}
        if func is not F.multi_head_attention_forward:
            return func(*args, **kwargs)
        assert kwargs.get("need_weights") is False, "the attention's dropout is only reached through SDPA with need_weights=False"
        saved = F.scaled_dot_product_attention
        F.scaled_dot_product_attention = self._sdpa
        try:
            return func(*args, **kwargs)
        finally:
            F.scaled_dot_product_attention = saved


def _run(m, ids, text, masks):
    """one forward + backward with every dropout replaced: masks None records the shapes, else applies them in order"""
    shapes, it = [], iter(masks or [])

    def take(x):
        if masks is None:
            shapes.append(tuple(x.shape))
            return x
        k = next(it)
        assert tuple(k.shape) == tuple(x.shape), (tuple(k.shape), tuple(x.shape))
        return x * k.to(x.dtype)

    for mod in m.modules():
        if isinstance(mod, torch.nn.Dropout):
            mod.forward = take
    m.zero_grad(set_to_none=True)
    with _Masks(take):
        out = m(ids, text)
        out.loss.backward()
    assert next(it, None) is None
    return out, shapes


def main(out=OUT):
    assert cobra_ref.available(), "reference tree not found"
    cfg = dict(cp.SMALL, decoder_dropout=P)
    torch.manual_seed(0)
    m = cobra_ref.ref_model(cfg, cp.cobra_params(cp.shapes(cfg), PARAM_SEED), dropout0=False)
    for mod in m.modules():                                   # the encoder's dropouts too (LightT5Encoder hard-codes 0.1)
        if isinstance(mod, torch.nn.Dropout):
            mod.p = P
        if isinstance(mod, torch.nn.MultiheadAttention):
            mod.dropout = P
    m = m.double().train()
    ids, text = cp.batch(cfg, seed=BATCH_SEED)
    _, shapes = _run(m, ids, text, None)
    res, _ = _run(m, ids, text, fixture_masks(shapes, MASK_SEED, P))
    fields = {k: getattr(res, k).detach().clone() for k in res._fields}
    vec_grads, sampled = {}, {}
    g = torch.Generator().manual_seed(7)
    for n, p in m.named_parameters():
        if p.dim() == 1:
            vec_grads[n] = p.grad.clone()
        else:
            pos = torch.randint(0, p.numel(), (SAMPLES,), generator=g)
            sampled[n] = dict(pos=pos.int(), values=p.grad.reshape(-1)[pos].clone(), frob=p.grad.norm().item())
    buf = io.BytesIO()
    torch.save(dict(cfg=cfg, param_seed=PARAM_SEED, batch_seed=BATCH_SEED, p=P, mask_seed=MASK_SEED, shapes=shapes, fields=fields,
                    vec_grads=vec_grads, sampled_grads=sampled), buf)
    with open(out, "wb") as f:
        f.write(buf.getvalue())
    print(out, os.path.getsize(out), "masks", len(shapes))


if __name__ == "__main__":
    main()
