"""COBRA without a GPU: the fp64 restatement (tests/cobra_reference.py) against the reference fixture, strict state_dict round
trips with the reference's Cobra, the new C symbols, and the refusals that come before any
launch."""
import ctypes
import os

import pytest
import torch

from tests import cobra_params as cp
from tests import cobra_reference as cr
from tests import cobra_ref

# measured worst errors of the fp64 restatement against the fp32 fixtures: fields 2.3e-7 (max-norm relative); gradients 4.8e-4
# (relative Frobenius: the encoder's gradients are about 1e-4 of the heads', so the fixture's own fp32 rounding shows there)
FP32_TOL = 4e-5
FP32_GRAD_TOL = 1e-3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, ref):
    return ((a.double() - ref.double()).abs().max() / ref.double().abs().max().clamp_min(1e-300)).item()


def _gerr(a, ref):
    return ((a.double() - ref.double()).norm() / ref.double().norm().clamp_min(1e-300)).item()


@pytest.mark.parametrize("name", ["cobra_small.pt", "cobra_trainer.pt"])
def test_restatement_matches_the_reference_fixture(golden, name):
    g = golden(name)
    cfg = g["cfg"]
    ids, text = cp.batch(cfg, seed=g["batch_seed"])
    out, grads = cr.step(cp.cobra_params(cp.shapes(cfg), g["param_seed"]), cfg, ids, text)
    for k, v in g["fields"].items():
        if v.is_floating_point():
            assert _rel(out[k], v) <= FP32_TOL, k
        else:
            assert out[k].item() == v.item(), k
    for n, v in g["vec_grads"].items():
        assert _gerr(grads[n], v) <= FP32_GRAD_TOL, n
    for n, s in g["sampled_grads"].items():
        assert _gerr(grads[n].reshape(-1)[s["pos"].long()], s["values"]) <= FP32_GRAD_TOL, n
        assert abs(grads[n].norm().item() - s["frob"]) <= FP32_GRAD_TOL * s["frob"], n
    assert set(g["vec_grads"]) | set(g["sampled_grads"]) == set(grads)


def test_restatement_equals_the_reference_under_dropout(golden):
    """cobra_small_dropout.pt: the reference's step in fp64 at p = 0.3 everywhere on pre-drawn masks; the masked restatement on the
    same masks matches it to 1e-10"""
    g = golden("cobra_small_dropout.pt")
    cfg = g["cfg"]
    ids, text = cp.batch(cfg, seed=g["batch_seed"])
    masks = cr.fixture_masks(g["shapes"], g["mask_seed"], g["p"])
    assert len(masks) == 4 + 5 * cfg["decoder_n_layers"] and all(bool((k == 0).any()) for k in masks)
    out, grads = cr.step(cp.cobra_params(cp.shapes(cfg), g["param_seed"]), cfg, ids, text, masks=masks)
    for k, v in g["fields"].items():
        if v.is_floating_point():
            # codebook_entropy: the reference counts the ids' usage in fp32 whatever the model's dtype
            assert _rel(out[k], v) <= (FP32_TOL if k == "codebook_entropy" else 1e-10), k
        else:
            assert out[k].item() == v.item(), k
    for n, v in g["vec_grads"].items():
        assert _rel(grads[n], v) <= 1e-10, n
    for n, s in g["sampled_grads"].items():
        a = grads[n].reshape(-1)[s["pos"].long()]
        assert (a - s["values"]).abs().max().item() <= 1e-10 * s["frob"], n
        assert abs(grads[n].norm().item() - s["frob"]) <= 1e-10 * s["frob"], n
    for bad in (masks[:-1], masks + masks[-1:]):                 # one mask short, one too many
        with pytest.raises(ValueError, match="masks than"):
            cr.step(cp.cobra_params(cp.shapes(cfg), g["param_seed"]), cfg, ids, text, masks=bad)


@pytest.mark.skipif(not cobra_ref.available(), reason="the reference tree is not present")
def test_the_dropout_fixture_regenerates_byte_for_byte(tmp_path):
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_cobra_dropout", os.path.join(ROOT, "scripts", "make_golden_cobra_dropout.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    out = tmp_path / "cobra_small_dropout.pt"
    mod.main(str(out))
    with open(os.path.join(ROOT, "tests", "golden", "cobra_small_dropout.pt"), "rb") as f:
        assert out.read_bytes() == f.read()


@pytest.mark.skipif(not cobra_ref.available(), reason="the reference tree is not present")
@pytest.mark.parametrize("cfg", [cp.SMALL, cp.TRAINER], ids=["small", "trainer"])
def test_state_dict_round_trips_strictly(cfg):
    from genrec_b200.cobra import Cobra
    ours = Cobra(**cfg)
    ref = cobra_ref.ref_model(cfg, ours.state_dict())
    ours.load_state_dict(ref.state_dict(), strict=True)
    assert {k: tuple(v.shape) for k, v in ours.state_dict().items()} == {k: tuple(v.shape) for k, v in ref.state_dict().items()}


def test_new_symbols_are_declared_and_bound():
    from genrec_b200 import _lib
    names = ["grb_post_layernorm_forward", "grb_post_layernorm_backward", "grb_cobra_pack_texts", "grb_cobra_text_rows", "grb_seg_layernorm_mean_forward", "grb_seg_layernorm_mean_backward",
             "grb_seg_layernorm_mean_backward_workspace_bytes", "grb_l2norm_forward", "grb_l2norm_backward",
             "grb_infonce_forward_backward"]
    header = open(os.path.join(ROOT, "include", "genrec_b200.h")).read()
    for n in names:
        assert n + "(" in header, n
        assert n in _lib.SIGNATURES, n
    if os.path.exists(_lib.LIB_PATH):
        lib = ctypes.CDLL(_lib.LIB_PATH)
        for n in names:
            assert hasattr(lib, n), n


def test_unsupported_shapes_raise_before_anything_runs():
    from genrec_b200 import _lib
    from genrec_b200.cobra import Cobra
    with pytest.raises(_lib.GrbError):
        Cobra(encoder_hidden_dim=768, encoder_num_heads=6)           # head dim 128
    with pytest.raises(_lib.GrbError):
        Cobra(d_model=384, decoder_num_heads=4)                       # head dim 96 in the decoder
    m = Cobra(**cp.SMALL)
    for name in ("generate", "beam_fusion"):
        with pytest.raises(NotImplementedError):
            getattr(m, name)()
