"""Write the COBRA reference fixtures from the reference's unmodified Cobra (genrec/models/cobra.py) on the CPU in fp32, every dropout
p set to 0 on the instance (the encoder's included), on the ragged batch of tests/cobra_params.py (users of 1, 2, 7 and 20 items;
texts of 1, 37 and 128 tokens; all-zero pad-item texts):

    tests/golden/cobra_small.pt                          encoder 192 (2 heads of 96), d_model 128, 2 decoder layers
    tests/golden/cobra_trainer.pt (+ .sampled_grads.pt)  the trainer's shape (genrec/trainers/cobra_trainer.py:92-135), B = 4

Each holds every CobraOutput field, every vector gradient and 1,024 seeded entries (plus the norm) of every matrix gradient of one
step.  The parameters are not stored: the tests rebuild them from (shapes, param_seed).  The seeds are searched until every counted
position's top-1 and top-5 logits lead the next class by at least MARGIN, so the integer metrics (acc_*, recall_*) of a bf16 model
can be compared exactly."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_loader  # noqa: E402
from tests import cobra_params as cp  # noqa: E402
from tests import cobra_ref  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
SAMPLES = 1024
# logit units; the heads' logits are about N(0, 1) plus the spread biases (cobra_params.HEAD_BIAS_STD), and their bf16 error is
# a few thousandths
MARGIN = 5e-2
TRIES = 200


def margins(m, ids, text, cfg):
    """(smallest top-1 lead, smallest top-5 lead) over the positions the metrics count, from the sparse heads' logits"""
    logs = []
    hooks = [h.register_forward_hook(lambda mod, i, o: logs.append(o.detach())) for h in m.sparse_head]
    try:
        with torch.no_grad():
            m(ids, text)
    finally:
        for h in hooks:
            h.remove()
    C, V = cfg["n_codebooks"], cfg["id_vocab_size"]
    T = ids.shape[1] // C
    g1 = g5 = float("inf")
    for c, lg in enumerate(logs):
        ok = ids[:, torch.arange(1, T) * C + c] != V * C
        top = lg[ok].topk(6, -1).values
        g1 = min(g1, (top[:, 0] - top[:, 1]).min().item())
        g5 = min(g5, (top[:, 4] - top[:, 5]).min().item())
    return g1, g5


def fixture(name, cfg, first_seed):
    shapes = cp.shapes(cfg)
    for k in range(TRIES):
        param_seed = batch_seed = first_seed + k
        P = cp.cobra_params(shapes, param_seed)
        ids, text = cp.batch(cfg, seed=batch_seed)
        m = cobra_ref.ref_model(cfg, P)
        g1, g5 = margins(m, ids, text, cfg)
        if min(g1, g5) >= MARGIN:
            break
    else:
        raise RuntimeError(f"{name}: no seed with the required margin")
    print(name, "seed", param_seed, "margins", g1, g5)
    out = m(ids, text)
    out.loss.backward()
    fields = {k: getattr(out, k).detach().clone() for k in out._fields}
    vec_grads, sampled = {}, {}
    g = torch.Generator().manual_seed(7)
    for n, p in m.named_parameters():
        if p.dim() == 1:
            vec_grads[n] = p.grad.clone()
        else:
            pos = torch.randint(0, p.numel(), (SAMPLES,), generator=g)
            sampled[n] = dict(pos=pos.int(), values=p.grad.reshape(-1)[pos].clone(), frob=p.grad.norm().item())
    head = dict(cfg=cfg, param_seed=param_seed, batch_seed=batch_seed, margins=(g1, g5), fields=fields, vec_grads=vec_grads)
    if name == "cobra_small":
        torch.save(dict(head, sampled_grads=sampled), os.path.join(OUT, name + ".pt"))
    else:                                            # two parts, each under 1 MB (tests/conftest.py joins them)
        torch.save(head, os.path.join(OUT, name + ".pt"))
        torch.save(sampled, os.path.join(OUT, name + ".sampled_grads.pt"))


def main():
    assert ref_loader.available(), "reference tree not found"
    fixture("cobra_small", dict(cp.SMALL), 100)
    fixture("cobra_trainer", dict(cp.TRAINER), 300)
    for f in sorted(os.listdir(OUT)):
        if f.startswith("cobra_"):
            print(f, os.path.getsize(os.path.join(OUT, f)))


if __name__ == "__main__":
    main()
