"""The HSTU block's feed-forward (hstu_ffn.cuh at D = 64 and 128, the four tc_gemm_kernel launches at D = 256) against the library's
unfused linear kernels, bit for bit, on the H100.

One block forward and backward through grb_hstu_layer_forward_jagged / _backward_jagged; then z1, hact and y are recomputed from
the block's own xn and x1 by grb_linear_forward + grb_linear_residual_forward, and dz1 and dxn from its dyb and saved z1 by
grb_linear_dact_backward + grb_linear_backward, with the block's dropout keys (site 8 layer + 1 and + 2, the same seed and seed_dev).
Every one must be torch.equal.  The row counts sit at the fused kernel's tile edges (64-row warpgroup halves, 128-row tiles) and
its persistent grid's edges (132 * 128 +- 1), plus the cfg2 batch and a packed batch with idle rows."""
import pytest
import torch

from tests.hstu_block_reference import site
from tests.hstu_cases import run_block_jagged

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

# (lengths, idle rows): T = sum(lengths) + idle
ROWS = {
    "T1": ([1], 0), "T63": ([63], 0), "T64": ([64], 0), "T65": ([65], 0), "T127": ([127], 0), "T128": ([128], 0),
    "T129": ([129], 0), "T16895": ([200] * 84 + [95], 0), "T16897": ([200] * 84 + [97], 0), "T25600": ([200] * 128, 0),
    "packed_idle": ([37, 150, 1, 80, 200], 5),
}
DROP = {"p0": (0.0, None), "p0.2": (0.2, None), "p0.2_seed_dev": (0.2, 12345)}


@pytest.mark.parametrize("drop", sorted(DROP))
@pytest.mark.parametrize("rows", sorted(ROWS))
@pytest.mark.parametrize("D", [64, 128, 256])
def test_ffn_matches_unfused_kernels(D, rows, drop):
    import genrec_b200.functional as Fn
    lengths, idle = ROWS[rows]
    p, seed_dev = DROP[drop]
    layer = 1
    r = run_block_jagged(lengths, D, D // 32, ("uni", 3), "nots", idle=idle, p=p, layer=layer, seed_dev=seed_dev)
    prm = r["prm"]
    seed = 0x1234_5678_9ABC_DEF0 + layer
    sdev = None if seed_dev is None else torch.tensor([seed_dev], dtype=torch.int64, device=DEV)
    hid, out = site(layer, 1), site(layer, 2)
    z1, hact = Fn.linear_fwd(r["xn"], prm["ffn1_w"], prm["ffn1_b"], 1, p, seed, sdev, hid)
    y = Fn.linear_residual_fwd(r["hact"], prm["ffn2_w"], prm["ffn2_b"], r["x1"], None, p, seed, sdev, out)
    dz1 = Fn.linear_dact_bwd(r["dyb"], prm["ffn2_w"], r["z1"], 1, p, seed, sdev, hid)
    dxn = Fn.linear_bwd(r["dz1"], prm["ffn1_w"], r["xn"], need_dw=False)[0]
    torch.cuda.synchronize()
    bad = [n for n, got, ref in (("z1", r["z1"], z1), ("hact", r["hact"], hact), ("y", r["y"], y), ("dz1", r["dz1"], dz1),
                                 ("dxn", r["dxn"], dxn)) if not torch.equal(got, ref)]
    assert not bad, f"not bit-identical to the unfused kernels: {bad}"
