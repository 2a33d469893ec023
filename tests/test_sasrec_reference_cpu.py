"""tests/sasrec_reference.py on the CPU: with every mask 1 it computes what the dropout-free oracle (oracle/sasrec.py) computes, loss,
logits and every gradient; its packed form computes, row by row, what its padded form computes on the same users left-padded under
the same masks; and the kernels' masks it restates have the shapes its forward consumes and drop at every site."""
import pytest
import torch

from oracle import sasrec as osr
from tests import sasrec_reference as sr
from tests.attention_reference import keep_scale

CFG = dict(num_items=97, max_seq_len=24, embed_dim=64, num_heads=2, num_blocks=2, ffn_dim=96)
LENGTHS = [5, 0, 24, 1, 17, 3, 24, 9]            # a user without history, one of a single item, two at the longest


def _rel(a, ref, floor=1e-300):
    """max-norm relative error; floor: the scale below which an entry counts as zero"""
    return ((a.double() - ref.double()).abs().max() / ref.double().abs().max().clamp_min(floor)).item()


def _grads_agree(got, ref):
    """every gradient to 1e-10 of itself, or of the largest gradient entry: d loss / d k_proj.bias is analytically zero (a shift
    of each query's scores by a constant cancels in the softmax), so it holds rounding noise alone"""
    assert set(got) == set(ref)
    top = max(v.abs().max().item() for v in ref.values())
    bad = {k: _rel(got[k], v, top) for k, v in ref.items() if _rel(got[k], v, 1e-6 * top) > 1e-10}
    assert not bad, bad


def _users(lengths, seed):
    g = torch.Generator().manual_seed(seed)
    hist = [torch.randint(1, CFG["num_items"] + 1, (n,), generator=g) for n in lengths]
    tgt = [torch.randint(1, CFG["num_items"] + 1, (n,), generator=g) for n in lengths]
    if len(hist[0]) > 2:
        hist[0][2] = 0                            # an id-0 token inside a history
    return hist, tgt


def _padded(hist, tgt):
    L = max(len(h) for h in hist)
    ids = torch.zeros(len(hist), L, dtype=torch.int64)
    tg = torch.zeros_like(ids)
    for b, (h, t) in enumerate(zip(hist, tgt)):
        if len(h):
            ids[b, L - len(h):], tg[b, L - len(h):] = h, t
    return {"input_ids": ids, "targets": torch.where(ids == 0, 0, tg)}


def _packed(hist, tgt, idle):
    offs = [0]
    for h in hist:
        offs.append(offs[-1] + len(h))
    ids = torch.cat([*hist, torch.randint(1, CFG["num_items"] + 1, (idle,))])   # idle rows holding real ids still give x = 0
    tg = torch.cat([*tgt, torch.zeros(idle, dtype=torch.int64)])
    return {"input_ids": ids, "targets": torch.where(ids == 0, 0, tg), "offsets": offs}


def test_all_ones_masks_equal_the_oracle():
    prm = {k: v.double() for k, v in sr.seeded_params(CFG, 1).items()}
    batch = _padded(*_users(LENGTHS, 2))
    B, L = batch["input_ids"].shape
    r = sr.step(prm, CFG, batch, sr.ones_masks(CFG, ("padded", B, L)))
    op = {k: v.clone().requires_grad_(True) for k, v in prm.items()}
    logits, loss = osr.sasrec_forward(batch["input_ids"], batch["targets"], op, CFG["num_heads"], CFG["num_blocks"])
    loss.backward()
    assert _rel(r["logits"], logits.detach()) <= 1e-12
    assert abs(r["loss"].item() - loss.item()) <= 1e-12 * abs(loss.item())
    grads = {k: v.grad for k, v in op.items() if v.grad is not None}
    assert set(grads) == set(prm)
    _grads_agree(r["grads"], grads)
    # no masks at all is the same step
    r0 = sr.step(prm, CFG, batch)
    assert torch.equal(r0["logits"], r["logits"])


@pytest.mark.parametrize("p", [0.2, 0.5])
def test_packed_form_equals_the_padded_form(p):
    """the same users left-padded and packed (with idle rows after them) under the same masks: every real row's logits, the loss and
    every gradient agree"""
    prm = sr.seeded_params(CFG, 3)
    hist, tgt = _users(LENGTHS, 4)
    pb, pk = _padded(hist, tgt), _packed(hist, tgt, idle=7)
    B, L = pb["input_ids"].shape
    T = pk["input_ids"].numel()
    D, H, ffn = CFG["embed_dim"], CFG["num_heads"], CFG["ffn_dim"]
    g = torch.Generator().manual_seed(int(10 * p))
    _, sc = keep_scale(p)
    drawn = lambda *shape: torch.where(torch.rand(*shape, generator=g) >= p, sc, 0.0).double()
    mp = {"emb": drawn(B * L, D), "attn": [drawn(B, H, L, L) for _ in range(2)], "hid": [drawn(B * L, ffn) for _ in range(2)],
          "out": [drawn(B * L, D) for _ in range(2)]}
    offs = pk["offsets"]
    rows = torch.tensor([b * L + L - len(h) + i for b, h in enumerate(hist) for i in range(len(h))])   # packed row -> padded row
    gather = lambda m, n: torch.cat([m[rows], torch.ones(T - len(rows), n, dtype=torch.float64)])
    mk = {"emb": gather(mp["emb"], D), "hid": [gather(m, ffn) for m in mp["hid"]], "out": [gather(m, D) for m in mp["out"]],
          "attn": [[a[b:b + 1, :, L - n:, L - n:] for b, n in enumerate(len(h) for h in hist)] for a in mp["attn"]]}
    rp = sr.step(prm, CFG, pb, mp)
    rk = sr.step(prm, CFG, pk, mk, packed=True)
    real = pb["input_ids"].reshape(-1) != 0
    live = torch.zeros(T, dtype=torch.bool)
    live[:offs[-1]] = pk["input_ids"][:offs[-1]] != 0
    assert _rel(rk["logits"][live], rp["logits"].reshape(B * L, -1)[real]) <= 1e-12
    assert abs(rk["loss"].item() - rp["loss"].item()) <= 1e-12 * abs(rp["loss"].item())
    _grads_agree(rk["grads"], rp["grads"])
    # the idle rows and id-0 rows are x = 0: their logits are the final norm's bias against the table
    zero = prm["final_norm.bias"].double() @ prm["item_embedding.weight"].double().T
    assert _rel(rk["logits"][~live], zero.expand(int((~live).sum()), -1)) <= 1e-12


@pytest.mark.parametrize("shape", [("padded", 8, 24), ("packed", 90, [0, 5, 5, 29, 30, 47, 50, 74, 83])])
def test_kernel_masks_fit_the_forward_and_drop_everywhere(shape):
    cfg = dict(CFG)
    m = sr.kernel_step_masks(cfg, 0.5, 0x1234_5678_9ABC, 977, shape)
    names = [n for n, _ in sr.mask_sources(m)]
    assert names == ["emb", "attn 0", "hid 0", "out 0", "attn 1", "hid 1", "out 1"]
    for n, k in sr.mask_sources(m):
        assert bool((k == 0).any()) and bool((k != 0).any()), n
    # another device seed value moves every mask
    m2 = sr.kernel_step_masks(cfg, 0.5, 0x1234_5678_9ABC, 978, shape)
    for (n, a), (_, b) in zip(sr.mask_sources(m), sr.mask_sources(m2)):
        assert not torch.equal(a, b), n
    T = shape[1] * shape[2] if shape[0] == "padded" else shape[1]
    ids = torch.randint(1, cfg["num_items"] + 1, (T,))
    batch = {"input_ids": ids.view(shape[1], shape[2]) if shape[0] == "padded" else ids, "targets": ids.roll(1).view(*(
        (shape[1], shape[2]) if shape[0] == "padded" else (T,)))}
    if shape[0] == "packed":
        batch["offsets"] = shape[2]
        batch["targets"][shape[2][-1]:] = 0
    r = sr.step(sr.seeded_params(cfg, 5), cfg, batch, m, packed=shape[0] == "packed")
    assert torch.isfinite(r["loss"])


def test_a_mask_of_the_wrong_shape_is_refused():
    batch = _padded(*_users(LENGTHS, 6))
    B, L = batch["input_ids"].shape
    m = sr.ones_masks(CFG, ("padded", B, L))
    m["hid"][1], m["out"][1] = m["out"][1], m["hid"][1]
    with pytest.raises(ValueError):
        sr.step(sr.seeded_params(CFG, 1), CFG, batch, m)
