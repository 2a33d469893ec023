"""Host-side checks of the paged serving pool (no GPU): the workspace query of grb_hstu_layer_extend_paged and the refusals of the
pool entry points, and the Python-side argument checks of HSTUPool."""
import ctypes

import pytest


@pytest.fixture(scope="module")
def lib():
    from genrec_b200 import build
    build.build()
    from genrec_b200 import _lib
    return _lib.load()


def _pool(page_size=64, max_items=256, max_users=8, num_pages=16, num_layers=2):
    from genrec_b200._lib import HstuPool
    return HstuPool(max_users, num_layers, page_size, num_pages, max_items, None, None, None, None, None, None, None, None, None)


def test_paged_workspace_bytes(lib):
    from genrec_b200._lib import HstuDims
    d = HstuDims(128, 1, 128, 4, 32, 64, 0.0, 0, None, 0)
    ws = lib.grb_hstu_layer_extend_paged_workspace_bytes(ctypes.byref(d), ctypes.byref(_pool(max_items=256)))
    # the same scratch as the dense cache of capacity max_items: the key split depends on the shapes and max_items only
    assert ws == lib.grb_hstu_layer_extend_workspace_bytes(ctypes.byref(d), 256) > 0
    assert lib.grb_hstu_layer_extend_paged_workspace_bytes(ctypes.byref(d), ctypes.byref(_pool(max_items=4096))) >= ws


@pytest.mark.parametrize("kw,msg", [(dict(page_size=96), b"page_size"), (dict(page_size=0), b"page_size"),
                                    (dict(page_size=32), b"page_size"), (dict(max_items=0), b"max_items"),
                                    (dict(max_items=16385), b"max_items"), (dict(max_users=0), b"pool shape"),
                                    (dict(num_pages=0), b"pool shape")])
def test_pool_refusals(lib, kw, msg):
    from genrec_b200._lib import HstuDims, HstuLayerParams
    d = HstuDims(4, 1, 128, 4, 32, 64, 0.0, 0, None, 0)
    pool = _pool(**kw)
    assert lib.grb_hstu_layer_extend_paged_workspace_bytes(ctypes.byref(d), ctypes.byref(pool)) == 0
    assert msg in lib.grb_last_error(), lib.grb_last_error()
    # every entry point refuses before touching any pointer
    rc = lib.grb_hstu_pool_append(ctypes.byref(pool), None, 4, None, None, 1, None, None, None, None)
    assert rc == -1 and msg in lib.grb_last_error()
    rc = lib.grb_hstu_pool_release(ctypes.byref(pool), None, 4, None, 0, None)
    assert rc == -1 and msg in lib.grb_last_error()
    rc = lib.grb_hstu_layer_extend_paged(ctypes.byref(d), ctypes.byref(HstuLayerParams()), ctypes.byref(pool), 0, None, None, None, 0, None,
                                         None, None, None, None)
    assert rc == -1 and msg in lib.grb_last_error()


def test_null_pointers_and_shapes(lib):
    from genrec_b200._lib import HstuDims, HstuLayerParams
    pool = _pool()
    assert lib.grb_hstu_layer_extend_paged_workspace_bytes(ctypes.byref(HstuDims(4, 1, 128, 4, 32, 64, 0.0, 0, None, 0)), None) == 0
    assert b"null pool" in lib.grb_last_error()
    assert lib.grb_hstu_pool_append(None, None, 4, None, None, 1, None, None, None, None) == -1
    assert b"null pool" in lib.grb_last_error()
    assert lib.grb_hstu_pool_append(ctypes.byref(pool), None, 4, None, None, 1, None, None, None, None) == -1
    assert b"null argument" in lib.grb_last_error()
    assert lib.grb_hstu_pool_release(ctypes.byref(pool), None, 4, None, 0, None) == -1
    assert b"null argument" in lib.grb_last_error()
    d = HstuDims(4, 1, 128, 4, 32, 64, 0.0, 0, None, 0)
    rc = lib.grb_hstu_layer_extend_paged(ctypes.byref(d), ctypes.byref(HstuLayerParams()), ctypes.byref(pool), 0, None, None, None, 0, None,
                                         None, None, None, None)
    assert rc == -1 and b"null argument" in lib.grb_last_error()
    # the dims are checked as for the dense cache: dropout, head_dim, B * ceil(n / 64)
    for bad, msg in ((HstuDims(4, 1, 128, 4, 32, 64, 0.1, 0, None, 0), b"dropout_p"), (HstuDims(4, 1, 96, 3, 32, 64, 0.0, 0, None, 0), b"unsupported"),
                     (HstuDims(65536, 1, 128, 4, 32, 64, 0.0, 0, None, 0), b"65535")):
        assert lib.grb_hstu_layer_extend_paged_workspace_bytes(ctypes.byref(bad), ctypes.byref(pool)) == 0
        assert msg in lib.grb_last_error(), lib.grb_last_error()


def test_python_pool_arguments():
    from genrec_b200.hstu import HSTUPool
    for kw, msg in ((dict(page_size=100), "page_size"), (dict(max_items=20000), "max_items"), (dict(max_users=0), "positive")):
        args = dict(max_users=4, num_pages=8, page_size=64, max_items=256, num_layers=1, embed_dim=64, device="cpu")
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            HSTUPool(**args)
