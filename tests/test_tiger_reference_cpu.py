"""tests/tiger_reference.py against the reference Tiger, on the CPU: with the dropout masks of tiger_small_dropout.pt (drawn at p = 0.3
and applied at every nn.Dropout of the reference) it computes the reference's fp64 step, which pins where every dropout sits; at
p = 0 it matches the fp32 reference fixtures; and its packed form computes, user by user, what its padded form computes."""
import pytest
import torch

from tests import tiger_params as tp
from tests import tiger_reference as tr
from tests.attention_reference import keep_scale

# measured worst relative error of the fp64 restatement against the fp32 reference fixtures (max-norm over each tensor): 8.2e-7
# (tiger_small.pt, user_id_embedding.emb.weight's gradient) and 3.9e-6 (tiger_published.pt, an encoder rel_bias gradient); the
# bound is ~10x the larger
FP32_TOL = 4e-5


def _params(g):
    return tp.tiger_params(g["shapes"], g["param_seed"])


def _rel(a, ref):
    """max-norm relative error"""
    return ((a.double() - ref.double()).abs().max() / ref.double().abs().max().clamp_min(1e-300)).item()


def test_restatement_equals_the_reference_under_dropout(golden):
    g = golden("tiger_small_dropout.pt")
    cfg = g["cfg"]
    masks = [k.double() * keep_scale(g["p"])[1] for k in g["keep"]]
    r = tr.step(_params(g), cfg, tp.batch(cfg, g["B"], g["n_items"], g["batch_seed"]), masks)
    assert _rel(r["logits"], g["logits"]) <= 1e-10
    assert abs(r["loss"].item() - g["loss"].item()) <= 1e-10 * abs(g["loss"].item())
    ref = {k: v for k, v in g.items() if k.startswith("grads")}
    grads = dict(ref.pop("grads"))
    for part in ref.values():
        grads.update(part)
    assert set(r["grads"]) == set(grads)
    for n, t in grads.items():
        assert _rel(r["grads"][n], t) <= 1e-10, n


def test_the_fixture_masks_drop_at_every_site(golden):
    """30 % of each mask dropped, within the binomial spread of its size: every dropout of the reference was reached"""
    g = golden("tiger_small_dropout.pt")
    assert len(g["keep"]) == 2 + 4 + 6                        # two input dropouts, one encoder and one decoder block
    for k in g["keep"]:
        frac = 1 - k.double().mean().item()
        assert abs(frac - g["p"]) < 5 * (g["p"] * (1 - g["p"]) / k.numel()) ** 0.5, (tuple(k.shape), frac)


def test_a_missing_or_extra_mask_is_refused(golden):
    g = golden("tiger_small_dropout.pt")
    cfg = g["cfg"]
    masks = [k.double() for k in g["keep"]]
    b = tp.batch(cfg, g["B"], g["n_items"], g["batch_seed"])
    with pytest.raises(ValueError):
        tr.step(_params(g), cfg, b, masks[:-1])
    with pytest.raises(ValueError):
        tr.step(_params(g), cfg, b, masks + masks[-1:])
    with pytest.raises(ValueError):
        tr.step(_params(g), cfg, b, masks[1:] + masks[:1])


def test_restatement_matches_the_fp32_small_fixture(golden):
    g = golden("tiger_small.pt")
    cfg = g["cfg"]
    r = tr.step(_params(g), cfg, tp.batch(cfg, g["B"], g["n_items"], g["batch_seed"]))
    errs = {"logits": _rel(r["logits"], g["logits"]), "loss": _rel(r["loss"], g["loss"])}
    grads = dict(g["grads"])
    for k, v in g.items():
        if k.startswith("grads_"):
            grads.update(v)
    assert set(grads) == set(r["grads"])
    errs.update({n: _rel(r["grads"][n], t) for n, t in grads.items()})
    print("tiger_small.pt worst", max(errs.items(), key=lambda kv: kv[1]))
    assert max(errs.values()) <= FP32_TOL, errs


def test_restatement_matches_the_fp32_published_fixture(golden):
    g = golden("tiger_published.pt")
    cfg = g["cfg"]
    r = tr.step(_params(g), cfg, tp.batch(cfg, g["B"], g["n_items"], g["batch_seed"]))
    errs = {"logits": _rel(r["logits"], g["logits"]), "loss": _rel(r["loss"], g["loss"])}
    errs.update({n: _rel(r["grads"][n], t) for n, t in g["vec_grads"].items()})
    for n, s in g["sampled_grads"].items():
        errs[n] = _rel(r["grads"][n].reshape(-1)[s["pos"]], s["values"])
        assert abs(r["grads"][n].norm().item() - s["frob"]) <= FP32_TOL * s["frob"], n
    assert set(g["vec_grads"]) | set(g["sampled_grads"]) == set(r["grads"])
    print("tiger_published.pt worst", max(errs.items(), key=lambda kv: kv[1]))
    assert max(errs.values()) <= FP32_TOL, errs


@pytest.mark.parametrize("idle", [0, 5])
def test_packed_form_equals_the_padded_form(idle):
    """p = 0, SMALL: forward_jagged's layout (each user's row then its items, `idle` rows past offsets[B]) gives the padded step"""
    cfg = dict(tp.SMALL)
    B, n_items = 4, 5
    b = tp.batch(cfg, B, n_items, 2)
    lens = b["seq_mask"].sum(1)
    off = [0]
    for n in lens.tolist():
        off.append(off[-1] + n + 1)
    T = off[-1] + idle
    ids = torch.zeros(T, dtype=torch.int64)
    types = torch.zeros(T, dtype=torch.int64)
    for i in range(B):
        ids[off[i] + 1:off[i + 1]] = b["item_input_ids"][i, :lens[i]]
        types[off[i] + 1:off[i + 1]] = b["token_type_ids"][i, :lens[i]]
    pk = dict(user_input_ids=b["user_input_ids"].view(-1), item_input_ids=ids, token_type_ids=types,
              mem_offsets=torch.tensor(off), max_len=int(lens.max()) + 1, target_input_ids=b["target_input_ids"],
              target_token_type_ids=b["target_token_type_ids"])
    params = tp.tiger_params([(n, s) for n, s in _shapes(cfg)], 1)
    ref = tr.step(params, cfg, b)
    got = tr.step(params, cfg, pk, packed=True)
    assert _rel(got["logits"], ref["logits"]) <= 1e-12
    assert abs(got["loss"].item() - ref["loss"].item()) <= 1e-12 * abs(ref["loss"].item())
    assert set(got["grads"]) == set(ref["grads"])
    for n in ref["grads"]:
        assert _rel(got["grads"][n], ref["grads"][n]) <= 1e-12, n


def _shapes(cfg):
    from genrec_b200.tiger import Tiger
    return [(k, tuple(v.shape)) for k, v in Tiger(**cfg).state_dict().items()]
