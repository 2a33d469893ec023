"""TEST INFRASTRUCTURE - the reference's unmodified genrec/models/cobra.py (build container only: the reference tree is not on the
GPU machines).  Its imports reach ``transformers`` (genrec/modules/encoder.py and, through genrec/__init__, the LLM models), which
is not installed, so an inert stub is registered first, next to the ``sentence_transformers`` stub of oracle/ref_loader.py: every
name imported from it (AutoTokenizer, AutoModel, T5EncoderModel, T5Config, ...) is an empty class."""
from __future__ import annotations

import sys
import types

from oracle import ref_loader


def available() -> bool:
    return ref_loader.available()


def _stub_class(name: str):
    if name.startswith("__"):
        raise AttributeError(name)
    return type(name, (), {})


def _install_transformers_stub() -> None:
    if "transformers" not in sys.modules:
        tf = types.ModuleType("transformers")
        tf.__getattr__ = _stub_class
        sys.modules["transformers"] = tf


def ref_cobra():
    """The reference's genrec.models.cobra module (Cobra, CobraOutput)."""
    _install_transformers_stub()
    return ref_loader._ref_module("genrec.models.cobra")


def ref_model(cfg: dict, params, dropout0: bool = True):
    """A reference Cobra with cfg's constructor arguments and the given state_dict; with dropout0 every dropout p is 0, the
    encoder's (which Cobra does not expose) included."""
    import torch
    import contextlib
    import io
    with contextlib.redirect_stdout(io.StringIO()):                 # LightT5Encoder prints on construction
        m = ref_cobra().Cobra(**cfg)
    m.load_state_dict(params, strict=True)
    if dropout0:
        for mod in m.modules():
            if isinstance(mod, torch.nn.Dropout):
                mod.p = 0.0
            if isinstance(mod, torch.nn.MultiheadAttention):
                mod.dropout = 0.0
    return m
