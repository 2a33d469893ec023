"""The C-ABI library loads on a CPU-only box and exports every symbol include/genrec_b200.h declares (no compute)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from genrec_b200 import build
    build.build()
    from genrec_b200 import _lib
    return _lib.load()


def test_every_declared_symbol_is_exported_and_bound(lib):
    from genrec_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "genrec_b200.h")).read()
    declared = set(re.findall(r"\b(grb_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations found"
    assert declared == set(_lib.SIGNATURES), (declared ^ set(_lib.SIGNATURES))
    for name in declared:
        assert hasattr(lib, name), name


def test_no_torch_types_in_the_abi():
    hdr = open(os.path.join(ROOT, "include", "genrec_b200.h")).read()
    assert "at::" not in hdr and "torch" not in hdr.replace("torch.optim.Adam", "").replace("no torch types", "")
    assert 'extern "C"' in hdr


def test_host_side_queries_and_errors(lib):
    from genrec_b200._lib import HstuDims
    assert lib.grb_version() >= 100
    d = HstuDims(128, 200, 128, 4, 32, 64, 0.0, 0, None, 0)
    T = 128 * 200
    saved = lib.grb_hstu_layer_saved_bytes(ctypes.byref(d))
    # xb, O, xn (bf16 [T,D]) + 4 x bf16 [T,4D] + x1 fp32 + 2 x stats
    assert saved >= T * 128 * 2 * 3 + T * 512 * 2 * 4 + T * 128 * 4 + 2 * T * 8
    assert lib.grb_hstu_layer_workspace_bytes(ctypes.byref(d)) > 0
    bad = HstuDims(1, 8, 96, 3, 32, 64, 0.0, 0, None, 0)
    assert lib.grb_hstu_layer_saved_bytes(ctypes.byref(bad)) == 0
    assert b"unsupported" in lib.grb_last_error()
    # D = 256 stores the [T, C] logits (bf16 gradient + fp32 logits); D <= 128 runs the fused kernels, which never form them
    assert lib.grb_head_workspace_bytes(T, 256, 12102) >= T * 12104 * (2 + 4)
    assert 0 < lib.grb_head_workspace_bytes(T, 128, 12102) < T * 12104 * 2


def test_product_never_imports_oracle():
    """The oracle is test infrastructure: nothing under genrec_b200/ or genrec/ may import it."""
    for pkg in ("genrec_b200", "genrec"):
        for dp, _, files in os.walk(os.path.join(ROOT, pkg)):
            for f in files:
                if f.endswith(".py"):
                    src = open(os.path.join(dp, f)).read()
                    assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), os.path.join(dp, f)


@pytest.mark.parametrize("B,L,D,H,refused", [
    (512, 65536, 64, 2, True),          # B L D = 2^31: the row offsets overflow int32
    (32768, 65536, 32, 1, True),        # B L H = 2^31: the dropout row key (b H + h) L + i overflows too
    (1801, 18631, 64, 2, False),        # B L D = 2^31 - 64: in range
])
def test_padded_sasrec_attention_refuses_rows_past_int32(lib, B, L, D, H, refused):
    """The padded SASRec attention entry points check B L H and B L D before anything else: a batch past int32 is refused with the
    bound, one inside it goes on to the next check (null pointers here, so nothing is launched and no memory is needed)."""
    from genrec_b200._lib import SasrecDims
    d = SasrecDims(B, L, D, H, 0.2, 1, None, 0)
    fwd = lib.grb_sasrec_attention_forward(ctypes.byref(d), *([None] * 7))
    fwd_msg = lib.grb_last_error()
    bwd = lib.grb_sasrec_attention_backward(ctypes.byref(d), *([None] * 11))
    bwd_msg = lib.grb_last_error()
    assert fwd != 0 and bwd != 0
    for msg in (fwd_msg, bwd_msg):
        assert (b"out of range" in msg) == refused, msg
        assert (b"null argument" in msg) == (not refused), msg
