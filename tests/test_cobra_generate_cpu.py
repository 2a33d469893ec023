"""COBRA generation without a GPU: the fp64 restatement (tests/cobra_generate_reference.py) against the reference fixture, the
fixture's regeneration, the new C symbols, and every refusal of generate / beam_fusion, which come before anything runs."""
import ctypes
import os

import pytest
import torch

from tests import cobra_generate_reference as gr
from tests import cobra_params as cp
from tests import cobra_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FP32_TOL = 1e-4            # fp64 restatement against the fp32 reference: scores and dense vectors, max-norm relative


def _rel(a, ref):
    return ((a.double() - ref.double()).abs().max() / ref.double().abs().max().clamp_min(1e-300)).item()


def _p64(cfg, seed):
    return {k: v.double() if v.is_floating_point() else v for k, v in gr.gen_params(cp.cobra_params(cp.shapes(cfg), seed)).items()}


def calls(cfg, seed):
    C = cfg["n_codebooks"]
    ids, text = cp.batch(cfg, seed=seed)
    out = [(f"user{b}", ids[b:b + 1, :n * C], text[b:b + 1, :n]) for b, n in enumerate(cp.ITEMS)]
    fids, ftext = cp.batch(cfg, items=(20, 20, 20), seed=seed + 1)
    return out + [("full", fids, ftext)]


@pytest.mark.parametrize("shape", ["small", "trainer"])
def test_restatement_matches_the_reference_fixture(golden, shape):
    g = golden("cobra_generate.pt")[shape]
    cfg = g["cfg"]
    P = _p64(cfg, g["param_seed"])
    for name, ids, text in calls(cfg, g["batch_seed"]):
        for K in (4, 20):
            ref = g["calls"][f"{name}_k{K}"]
            out = gr.generate(P, cfg, ids, text, K)
            assert torch.equal(out["sem_ids"], ref["sem_ids"]), (name, K)
            assert _rel(out["scores"], ref["scores"]) <= FP32_TOL, (name, K)
            assert _rel(out["dense_vecs"], ref["dense_vecs"]) <= FP32_TOL, (name, K)
    f = g["fusion"]
    _, fids, ftext = calls(cfg, g["batch_seed"])[-1]
    vecs, sem = gr.catalog(cfg, g["calls"]["full_k20"]["dense_vecs"][:, 0], f["catalog_seed"])
    out = gr.beam_fusion(P, cfg, fids, ftext, vecs.double(), sem, n_candidates=f["n_candidates"], n_beam=f["n_beam"],
                         temperature=f["temperature"], alpha=f["alpha"])
    assert torch.equal(out["item_ids"], f["item_ids"]) and torch.equal(out["sem_ids"], f["sem_ids"])
    assert (out["scores"] - f["scores"].double()).abs().max().item() <= 1e-5
    assert torch.allclose(out["leads"].float(), f["leads"]) and torch.allclose(out["sim_leads"].float(), f["sim_leads"])


@pytest.mark.skipif(not cobra_ref.available(), reason="the reference tree is not present")
def test_the_fixture_regenerates_byte_for_byte(tmp_path):
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_cobra_generate", os.path.join(ROOT, "scripts", "make_golden_cobra_generate.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    out = tmp_path / "cobra_generate.pt"
    mod.main(str(out))
    with open(os.path.join(ROOT, "tests", "golden", "cobra_generate.pt"), "rb") as f:
        assert out.read_bytes() == f.read()


def test_new_symbols_are_declared_and_bound():
    from genrec_b200 import _lib
    names = ["grb_cobra_beam_attention", "grb_cobra_beam_attention_workspace_bytes", "grb_cobra_beam_topk", "grb_cobra_beam_topk_workspace_bytes",
             "grb_cobra_dense_match", "grb_cobra_dense_match_workspace_bytes"]
    header = open(os.path.join(ROOT, "include", "genrec_b200.h")).read()
    for n in names:
        assert n + "(" in header, n
        assert n in _lib.SIGNATURES, n
    if os.path.exists(_lib.LIB_PATH):
        lib = ctypes.CDLL(_lib.LIB_PATH)
        for n in names:
            assert hasattr(lib, n), n


def test_the_output_types_are_exported():
    import genrec_b200.cobra as gc
    assert {"CobraGenerationOutput", "BeamFusionOutput"} <= set(gc.__all__)
    assert gc.CobraGenerationOutput._fields == ("sem_ids", "dense_vecs", "scores")
    assert gc.BeamFusionOutput._fields == ("item_ids", "sem_ids", "scores")


def test_missing_history_arguments_raise_a_type_error_that_names_them():
    from genrec_b200.cobra import Cobra
    m = Cobra(**cp.SMALL)
    with pytest.raises(TypeError, match="'encoder_input_ids'"):
        m.generate(torch.zeros(1, 3, dtype=torch.long))
    with pytest.raises(NotImplementedError, match="'item_dense_vecs', 'item_sem_ids'"):
        m.beam_fusion(torch.zeros(1, 3, dtype=torch.long), torch.zeros(1, 1, 4, dtype=torch.long))


def test_refusals_come_before_anything_runs():
    """CPU tensors: a call that passed its checks would stop at the CUDA requirement (RuntimeError), so every ValueError below comes
    from a check before any launch"""
    from genrec_b200.cobra import Cobra
    cfg = dict(cp.SMALL)
    m = Cobra(**cfg)
    C, V = cfg["n_codebooks"], cfg["id_vocab_size"]
    ids, text = cp.batch(cfg, items=(2, 3))
    D = cfg["d_model"]
    vecs, sem = torch.randn(5, D), torch.zeros(5, C, dtype=torch.long)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.generate(ids, text)
    for K in (0, V + 1, 1025):
        with pytest.raises(ValueError, match="n_candidates"):
            m.generate(ids, text, n_candidates=K)
    with pytest.raises(ValueError, match="n_candidates"):           # K V > 262,144 at V = 512, K = 513
        Cobra(**{**cfg, "id_vocab_size": 1024}).generate(ids, text, n_candidates=257)
    for t in (0.0, -1.0):
        with pytest.raises(ValueError, match="temperature"):
            m.generate(ids, text, temperature=t)
    empty = ids.clone()
    empty[0] = V * C
    with pytest.raises(ValueError, match="no item"):
        m.generate(empty, text)
    gap = ids.clone()
    gap[1, :C] = V * C                                              # a pad item before two real ones
    with pytest.raises(ValueError, match="follows a pad item"):
        m.generate(gap, text)
    T = -(-(cfg["max_len"] - C + 1) // (C + 1))                     # the fewest items with T (C+1) + C - 1 >= max_len
    long_ids, long_text = cp.batch(cfg, items=(T,), L=4)
    with pytest.raises(ValueError, match="max_len"):
        m.generate(long_ids, long_text)
    with pytest.raises(ValueError, match="encoder_input_ids"):
        m.generate(ids, text[:, :1])
    with pytest.raises(RuntimeError, match="CUDA"):
        m.beam_fusion(ids, text, vecs, sem, n_candidates=4, n_beam=8)
    for nc, nb in ((0, 8), (9, 8)):
        with pytest.raises(ValueError, match="n_candidates"):
            m.beam_fusion(ids, text, vecs, sem, n_candidates=nc, n_beam=nb)
    for nb in (V + 1, 1025):
        with pytest.raises(ValueError, match="n_beam"):
            m.beam_fusion(ids, text, vecs, sem, n_candidates=4, n_beam=nb)
    with pytest.raises(ValueError, match="item_dense_vecs"):
        m.beam_fusion(ids, text, torch.randn(5, D + 1), sem, n_candidates=4, n_beam=8)
    with pytest.raises(ValueError, match="item_sem_ids"):
        m.beam_fusion(ids, text, vecs, sem[:, :2], n_candidates=4, n_beam=8)
    with pytest.raises(ValueError, match="item_sem_ids"):
        m.beam_fusion(ids, text, vecs, sem[:4], n_candidates=4, n_beam=8)
    with pytest.raises(ValueError, match="temperature"):
        m.beam_fusion(ids, text, vecs, sem, n_candidates=4, n_beam=8, temperature=0.0)
