"""genrec_b200.tiger.Tiger without a device: the reference's parameter schema (recorded in tests/golden/tiger_*.pt), argument checks,
the shared parameter rebuild, and the genrec.models.tiger import path."""
import pytest
import torch

from tests import tiger_params as tp


@pytest.mark.parametrize("name", ["tiger_small.pt", "tiger_published.pt"])
def test_state_dict_schema_matches_the_reference(golden, name):
    from genrec_b200.tiger import Tiger
    g = golden(name)
    m = Tiger(**g["cfg"])
    got = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    assert got == [(k, tuple(s)) for k, s in g["shapes"]]
    m.load_state_dict(tp.tiger_params(g["shapes"], g["param_seed"]), strict=True)
    assert m.vocab_size == 769 if name == "tiger_published.pt" else m.vocab_size == 49


@pytest.mark.parametrize("kw", [dict(attn_dim=384, num_heads=8), dict(attn_dim=384, num_heads=3), dict(attn_dim=100, num_heads=2),
                                dict(embedding_dim=100), dict(embedding_dim=96), dict(attn_dim=512, num_heads=8)])
def test_bad_arguments_raise_before_any_launch(kw):
    from genrec_b200 import _lib
    from genrec_b200.tiger import Tiger
    cfg = dict(tp.PUBLISHED, **kw)
    with pytest.raises(_lib.GrbError):
        Tiger(**cfg)


def test_parameter_rebuild_is_deterministic():
    shapes = [("bos_embedding", (8,)), ("norm.weight", (8,)), ("sem_id_embedding.emb.weight", (7, 8)), ("a.rel_bias.weight", (64, 1)),
              ("in_proj.weight", (16, 8))]
    a, b = tp.tiger_params(shapes, 5), tp.tiger_params(shapes, 5)
    assert list(a) == [n for n, _ in shapes]
    for n in a:
        assert torch.equal(a[n], b[n]) and a[n].dtype == torch.float32
    assert not torch.equal(a["in_proj.weight"], tp.tiger_params(shapes, 6)["in_proj.weight"])
    assert (a["sem_id_embedding.emb.weight"][-1] == 0).all()               # the padding row
    x, y = tp.batch(tp.PUBLISHED, 4, 20, 9), tp.batch(tp.PUBLISHED, 4, 20, 9)
    for k in x:
        assert torch.equal(x[k], y[k])
    assert (x["seq_mask"][1:] == 0).any(dim=1).all()                        # every user but the first has padding


def test_genrec_models_tiger_still_resolves_to_the_reference(tmp_path, monkeypatch):
    """This repository provides no genrec.models.tiger: with a reference checkout on sys.path the reference module is found."""
    import importlib
    import os
    import sys
    ref = tmp_path / "refcheckout" / "genrec"
    (ref / "models").mkdir(parents=True)
    (ref / "__init__.py").write_text("")
    (ref / "models" / "tiger.py").write_text("MARK = 'reference tiger'\n")
    monkeypatch.syspath_prepend(str(tmp_path / "refcheckout"))
    for k in [k for k in sys.modules if k == "genrec" or k.startswith("genrec.")]:
        monkeypatch.delitem(sys.modules, k)
    monkeypatch.syspath_prepend(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    assert importlib.import_module("genrec.models.tiger").MARK == "reference tiger"
