"""fp64 references of the HSTU block's kernels - the gate (ln_gate_fwd_kernel / ln_gate_bwd_kernel), the cast of dy with the
FFN output bias gradient (cast_colsum_f32_bf16_kernel), the HSTU attention (csrc/attn_hstu.cuh) - of the wiring of the block's
linear layers (grb_hstu_layer_forward / _backward in csrc/api.cu) and of the fused Adam step (adam_tick_kernel + adam_step_kernel),
that know where the kernels round; and the fp64 rule of FlatAdam's lazy item-table step (lazy_adam_reference).

Each reference takes the kernel's own inputs to its stage (the bf16 P, zp, O, xn, hact and the saved LayerNorm statistics of the
forward's saved blob; dO, dxn, dx1, dyb, dz1 of the backward's workspace), so an error in one stage is not charged to the next and
each allowance is a bound derived from that stage alone.  The checks divide |got - ref| by the allowance; every allowance here is
derived, so the tolerance is dense_reference.TOL = 1, except where a comment quotes a measurement.

Where the kernels round (C = 2^-24 the fp32 unit roundoff, U = 2^-8 half a bf16 ulp, relative; SILU_SLACK the fast sigmoid):
  inputs            xb = RNE(x): bit for bit.
  projection        zp = bf16(x Wp^T + bp), P = bf16(silu(zp)): dense_reference.linear_forward.
  attention fwd     S = Q K^T is an fp32 sum of dh exact bf16 products (dh ACC |Q||K|); x = S + w with w = wpos[pb] + wtime[tb] the
                    fp32 table sum (restated exactly, `cell_bias`), one rounding C |x|; A = siluf(x) = x sigmoidf_fast(x): |silu'| <= 1.1
                    times the error of x plus SILU_SLACK |x| (1 + |x|); A is packed to bf16 (att_pack_p, U |A|); O = sum_j A_ij V_jd
                    in fp32 over at most L keys (L ACC per term), stored as bf16.  The allowance of O[i, d] is built from
                    sum_j (e_A + (U + L ACC) |A_ij|) |V_jd| of that element, not from the tensor's maximum.
  attention bwd     dA = dO V^T (dh ACC); dS = dA silu'(x): silu'' <= 1/2 times the error of x plus SILU_SLACK (1 + |x|) (dsiluf
                    in the dQ kernel and sg (1 + x (1 - sg)) in the dK/dV kernel are the same expression); dS and A are packed to
                    bf16; dQ = dS K, dK = dS^T Q, dV = A^T dO in fp32, times silu'(z) of the bf16 pre-activation (SILU_SLACK (1 + |z|)),
                    stored as bf16.  dpos / dtime keep the per-row bound of test_hstu_bias_configs_gpu (TABLE_C of each row's mass).
  gate fwd          N = LN1(O) two-pass on the bf16 O, g = N U (one product) times the keep scale of site 8 layer + 0 (row key =
                    token row, column c), x1 = x + g in fp32, xn = bf16(LN2(x1)); LN1 / LN2 carry dense_reference's row-sum depth
                    and large-offset terms.  st1 / st2 = (mean, rstd).
  gate bwd          from the saved st1 / st2: dx1 = dy + LN2bwd(dxn) (fp32, dense_reference.layernorm_backward with res = dy);
                    dG = dropmask(dx1); dzu = bf16(dG N silu'(zu)) into the U columns of dzp; dN = dG U; dO = bf16(LN1bwd(dN));
                    dg1, db1, dg2, db2 summed per warp, per CTA, then det_finish in order (T ACC per term).
  FFN               z1 / hact: linear_forward at site 8 layer + 1; y = x1 + drop(hact W2^T + b2) at site 8 layer + 2: linear_residual.
                    dyb = RNE(fp32(dy keep)) bit for bit; db2 = the column sums of dyb; dz1 = bf16(dropmask(dyb W2) silu'(z1))
                    (linear_dact_backward); dxn = dz1 W1; dx = dx1 + dzp Wp; db1 / bp the column sums of dz1 / dzp; dW2, dW1, dWp
                    linear_backward's dW bound.
  Adam              torch.optim.Adam in fp64 from the kernel's previous m, v, p and the fp32 hyper-parameters the ABI passes:
                    g = g0 grad_scale + wd p (L2 decay), m, v, bias corrections 1 - beta^t from the fp32 step counter; the library is
                    built with --use_fast_math, so powf is __powf (exp2 of y log2 x: 2^-22.5 absolute in log2 x, 2 ulp in exp2),
                    and the divisions and sqrtf are approximate (DIV per operation).  The bf16 mirror is RNE of the new fp32 p,
                    bit for bit; the gradient is exactly 0 afterwards when zero_grad is set.

Dropout masks are attention_reference.drop_mask (dense_reference.keep); with a non-null seed_dev the kernels add *seed_dev to the
seed (Dropout::resolve), `effective_seed` restates that.
"""
import math

import numpy as np
import torch

from tests.attention_reference import U, drop_mask, keep_scale
from tests.dense_reference import (ACC, C, RSQRT, SILU_SLACK, keep, layernorm_backward, layernorm_forward, linear_backward,
                                   linear_forward, linear_residual)

SITE_GATE, SITE_FFN_HID, SITE_FFN_OUT = 0, 1, 2       # csrc/api.cu: site = 8 layer + which
DIV = 2.0 ** -21                                      # approximate division / sqrtf under --use_fast_math: 4 ulp
LOG2_ABS = 2.0 ** -22.5                               # __log2f absolute error on [0.5, 2]
EXP2_REL = 2.0 ** -22                                 # __exp2f: 2 ulp
EPS = 1e-5                                            # the block's LayerNorm eps


def site(layer, which):
    return 8 * layer + which


def effective_seed(seed, p, seed_dev_value=None):
    """Dropout::resolve: with p > 0 and a seed_dev, the seed the kernels hash is seed + *seed_dev (mod 2^64)."""
    if p <= 0 or seed_dev_value is None:
        return seed
    return (seed + seed_dev_value) % (1 << 64)


def dsilu(z):
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s))


# ------------------------------------------------------------------------------------------------ carved layouts (csrc/api.cu)
def _align(n):
    return (n + 255) // 256 * 256


def saved_layout(T, D):
    """carve_saved: name -> (byte offset, dtype, shape); "bytes" the blob's size."""
    regions = [("xb", torch.bfloat16, (T, D)), ("zp", torch.bfloat16, (T, 4 * D)), ("P", torch.bfloat16, (T, 4 * D)),
               ("O", torch.bfloat16, (T, D)), ("st1", torch.float32, (T, 2)), ("x1", torch.float32, (T, D)),
               ("xn", torch.bfloat16, (T, D)), ("st2", torch.float32, (T, 2)), ("z1", torch.bfloat16, (T, 4 * D)),
               ("hact", torch.bfloat16, (T, 4 * D))]
    return _carve(regions)


def work_layout(T, D):
    """the first six regions of carve_work (the scratch of the ordered sums follows them); "bytes" the prefix's size."""
    regions = [("dyb", torch.bfloat16, (T, D)), ("dz1", torch.bfloat16, (T, 4 * D)), ("dxn", torch.float32, (T, D)),
               ("dx1", torch.float32, (T, D)), ("dO", torch.bfloat16, (T, D)), ("dzp", torch.bfloat16, (T, 4 * D))]
    return _carve(regions)


def _carve(regions):
    out, off = {}, 0
    for name, dt, shape in regions:
        out[name] = (off, dt, shape)
        off += _align(math.prod(shape) * torch.tensor([], dtype=dt).element_size())
    out["bytes"] = off
    return out


def view(blob, layout, name):
    off, dt, shape = layout[name]
    n = math.prod(shape) * torch.tensor([], dtype=dt).element_size()
    return blob[off:off + n].view(dt).view(shape)


# ------------------------------------------------------------------------------------------------ gate
def gate_forward(O, Uc, x, x1, g1, b1, g2, b2, p=0.0, seed=0, site_=0, eps=EPS):
    """O, Uc [T, D] bf16 (the kernel's O and the U columns of P), x [T, D] fp32, x1 the kernel's x1 (LN2's input).  -> "x1", "xn",
    "mean1", "rstd1", "mean2", "rstd2" with allowances, "drop" [T, D] (True = the gate's dropout drops)."""
    T, D = O.shape
    ln1 = layernorm_forward(O.float(), g1, b1, eps)
    km = keep(range(T), D, p, seed, site_, O.device)
    u = Uc.double()
    g = ln1["y"] * u * km
    a_g = (ln1["a_y32"] * u.abs() + 2 * C * (ln1["y"] * u).abs()) * km        # N's error, the product and the keep-scale product
    r = {"x1": x.double() + g, "drop": km == 0}
    r["a_x1"] = a_g + C * r["x1"].abs()
    ln2 = layernorm_forward(x1, g2, b2, eps)
    r.update(xn=ln2["y"], a_xn=ln2["a_y16"], mean1=ln1["mean"], a_mean1=ln1["a_mean"], rstd1=ln1["rstd"], a_rstd1=ln1["a_rstd"],
             mean2=ln2["mean"], a_mean2=ln2["a_mean"], rstd2=ln2["rstd"], a_rstd2=ln2["a_rstd"])
    return r


def gate_backward(dy, dxn, x1, st1, st2, O, Uc, zu, dx1, g1, b1, g2, p=0.0, seed=0, site_=0):
    """From the kernel's saved x1, st1, st2 and its own dx1 (the input of the gate half): -> "dx1", "dzu", "dO", "dg1", "db1", "dg2",
    "db2" with allowances."""
    T, D = O.shape
    r = {}
    b2w = layernorm_backward(dxn, x1, st2, g2, res=dy)
    r.update(dx1=b2w["dx"], a_dx1=b2w["a_dx"], dg2=b2w["dg"], a_dg2=b2w["a_dg"], db2=b2w["db"], a_db2=b2w["a_db"])
    km = keep(range(T), D, p, seed, site_, O.device)
    dG = dx1.double() * km
    st = st1.double()
    m1, r1 = st[:, 0:1], st[:, 1:2]
    o, u, z = O.double(), Uc.double(), zu.double()
    G1, B1 = g1.double(), b1.double()
    xh = (o - m1) * r1
    e_xh = 2 * C * (xh.abs() + r1 * o.abs())
    n = xh * G1 + B1
    a_n = G1.abs() * e_xh + 2 * C * ((G1 * xh).abs() + B1.abs())
    ds = dsilu(z)
    dzu = dG * n * ds
    a_dzu = dG.abs() * (a_n * ds.abs() + n.abs() * SILU_SLACK * (1 + z.abs())) + 3 * C * dzu.abs()
    r.update(dzu=dzu, a_dzu=U * dzu.abs() + (1 + U) * a_dzu)
    dN = dG * u                                                        # 2 C: the keep-scale product and this one
    b1w = layernorm_backward(dN, O.float(), st1, g1)
    gg = dN * G1
    extra = 2 * C * r1 * (gg.abs() + gg.abs().mean(1, keepdim=True) + xh.abs() * (gg * xh).abs().mean(1, keepdim=True))
    r.update(dO=b1w["dx"], a_dO=U * b1w["dx"].abs() + (1 + U) * (b1w["a_dx"] + extra))
    r.update(dg1=b1w["dg"], a_dg1=b1w["a_dg"] + 3 * C * (dN.abs() * (xh.abs() + e_xh)).sum(0),
             db1=b1w["db"], a_db1=b1w["a_db"] + 2 * C * dN.abs().sum(0))
    return r


def cast_colsum(dy, p=0.0, seed=0, site_=0):
    """dyb = RNE(fp32(dy keep)) (bit for bit: "dyb_exact"), "db" = the column sums of dyb with "a_db", "drop"."""
    T, D = dy.shape
    drop = torch.from_numpy(drop_mask(np.arange(T), D, p, seed, site_)).to(dy.device)
    sc = float(np.float32(keep_scale(p)[1]))
    dyb = torch.where(drop, torch.zeros_like(dy, dtype=torch.float32), dy.float() * sc).bfloat16()
    return {"dyb_exact": dyb, "db": dyb.double().sum(0), "a_db": T * ACC * dyb.double().abs().sum(0), "drop": drop}


def linear_dact_backward(dyb, w, z, p=0.0, seed=0, site_=0, act=1):
    """g = bf16(dropmask(dyb w) act'(z)) (TcEpiDAct<act>: 1 SiLU, 2 ReLU): dyb [T, K] bf16, w [K, N] bf16, z [T, N] bf16.
    -> "g", "a_g"."""
    DY, W, Z = dyb.double(), w.double(), z.double()
    T, K = DY.shape
    acc = DY @ W
    d = dsilu(Z) if act == 1 else (Z > 0).double()
    km = keep(range(T), W.shape[1], p, seed, site_, DY.device)
    g = acc * d * km
    slack = SILU_SLACK * acc.abs() * (1 + Z.abs()) if act == 1 else 0.0
    a = U * g.abs() + (K * ACC * (DY.abs() @ W.abs()) * d.abs() + slack) * km
    return {"g": g, "a_g": a}


# ------------------------------------------------------------------------------------------------ the row-wise stages of one block
def block_stage_items(r, seq=None):
    """Every stage of one block but the attention, each on the kernel's own inputs to it: projection, gate forward and backward, FFN,
    the cast of dy with its column sums, projection backward.  r: the inputs, intermediates and gradients of one forward + backward
    (x, y, dy, dx, grads, prm, p, layer, seed = the effective dropout seed, and the saved / workspace regions by name).  Asserts the
    bit-for-bit stages and the drop masks (x1 - x == 0 where the gate drops, hact == 0 where drop_hid drops).

    seq: None, or a bool [T] that is False on the idle rows of a packed batch (dy == 0 there).  The reference then takes the
    backward's intermediates dxn, dx1, dz1 and dzp as zero on the idle rows: the gradients of those rows are held to 0 and the column
    sums and weight gradients are the sums over the sequence rows alone.  -> [(name, got, ref, allowance)]"""
    p, layer, seed = r["p"], r["layer"], r["seed"]
    prm, gr, D = r["prm"], r["grads"], r["x"].shape[1]
    s_gate, s_hid, s_out = (site(layer, w) for w in (SITE_GATE, SITE_FFN_HID, SITE_FFN_OUT))
    live = (lambda t: t) if seq is None else (lambda t: torch.where(seq[:, None], t, torch.zeros((), dtype=t.dtype, device=t.device)))
    for n in ("xb", "zp", "P", "O", "st1", "x1", "xn", "st2", "z1", "hact", "dyb", "dz1", "dxn", "dx1", "dO", "dzp"):
        assert bool(torch.isfinite(r[n].float()).all()), f"{n} has an unwritten or non-finite element"
    assert torch.equal(r["xb"], r["x"].bfloat16()), "xb != RNE(x)"
    pj = linear_forward(r["xb"], prm["proj_w"], prm["proj_b"], 1, r["zp"])
    items = [("zp", r["zp"], pj["z"], pj["a_z"]), ("P", r["P"], pj["a"], pj["a_a"])]
    # gate forward
    Uc = r["P"][:, :D]
    gf = gate_forward(r["O"], Uc, r["x"], r["x1"], prm["ln1_g"], prm["ln1_b"], prm["ln2_g"], prm["ln2_b"], p, seed, s_gate)
    assert not bool((r["x1"] - r["x"])[gf["drop"]].any()), "x1 - x != 0 where the gate drops"
    items += [("x1", r["x1"], gf["x1"], gf["a_x1"]), ("xn", r["xn"], gf["xn"], gf["a_xn"]),
              ("st1 mean", r["st1"][:, 0], gf["mean1"], gf["a_mean1"]), ("st1 rstd", r["st1"][:, 1], gf["rstd1"], gf["a_rstd1"]),
              ("st2 mean", r["st2"][:, 0], gf["mean2"], gf["a_mean2"]), ("st2 rstd", r["st2"][:, 1], gf["rstd2"], gf["a_rstd2"])]
    # FFN forward
    f1 = linear_forward(r["xn"], prm["ffn1_w"], prm["ffn1_b"], 1, r["z1"], p, seed, s_hid)
    assert not bool(r["hact"][f1["a"] == 0].any()), "hact != 0 where drop_hid drops"
    f2 = linear_residual(r["hact"], prm["ffn2_w"], prm["ffn2_b"], r["x1"], None, p, seed, s_out)
    items += [("z1", r["z1"], f1["z"], f1["a_z"]), ("hact", r["hact"], f1["a"], f1["a_a"]), ("y", r["y"], f2["y"], f2["a_y"])]
    # backward: cast of dy, FFN, gate
    cc = cast_colsum(r["dy"], p, seed, s_out)
    assert torch.equal(r["dyb"], cc["dyb_exact"]), "dyb != RNE(fp32(dy keep))"
    if p in (0.0, 0.5):
        assert torch.equal(gr["ffn2_b"].double(), cc["db"]), "db2 is not the exact column sum of dyb"
    items.append(("dffn2_b", gr["ffn2_b"], cc["db"], cc["a_db"]))
    dz = linear_dact_backward(r["dyb"], prm["ffn2_w"], r["z1"], p, seed, s_hid)
    b1 = linear_backward(live(r["dz1"]), prm["ffn1_w"], r["xn"])
    b2 = linear_backward(r["dyb"], prm["ffn2_w"], r["hact"])
    items += [("dz1", r["dz1"], dz["g"], dz["a_g"]), ("dxn", r["dxn"], b1["dx"], b1["a_dx"]), ("dW1", gr["ffn1_w"], b1["dw"], b1["a_dw"]),
              ("dffn1_b", gr["ffn1_b"], b1["db"], b1["a_db"]), ("dW2", gr["ffn2_w"], b2["dw"], b2["a_dw"])]
    gb = gate_backward(r["dy"], live(r["dxn"]), r["x1"], r["st1"], r["st2"], r["O"], Uc, r["zp"][:, :D], live(r["dx1"]), prm["ln1_g"],
                       prm["ln1_b"], prm["ln2_g"], p, seed, s_gate)
    items += [("dx1", r["dx1"], gb["dx1"], gb["a_dx1"]), ("dzu", r["dzp"][:, :D], gb["dzu"], gb["a_dzu"]), ("dO", r["dO"], gb["dO"], gb["a_dO"]),
              ("dln1_g", gr["ln1_g"], gb["dg1"], gb["a_dg1"]), ("dln1_b", gr["ln1_b"], gb["db1"], gb["a_db1"]),
              ("dln2_g", gr["ln2_g"], gb["dg2"], gb["a_dg2"]), ("dln2_b", gr["ln2_b"], gb["db2"], gb["a_db2"])]
    # projection backward
    bp = linear_backward(live(r["dzp"]), prm["proj_w"], r["xb"], res=live(r["dx1"]))
    items += [("dx", r["dx"], bp["dx"], bp["a_dx"]), ("dWp", gr["proj_w"], bp["dw"], bp["a_dw"]), ("dproj_b", gr["proj_b"], bp["db"], bp["a_db"])]
    return items


# ------------------------------------------------------------------------------------------------ attention
def cell_bias(bias_index, wpos, wtime, npos_index, H):
    """Decode the [B, L, ld] index matrix the attention kernels read (pb * 64 + tb, sentinel npos_index * 64) into the fp32 table sum
    w [B, H, L, L] of att_build_table and the masked cells [B, 1, L, L].  wpos [rows, H] (the live row alone when the buckets are
    uniform), wtime [ntime, H] or None (then no time term)."""
    B, L = bias_index.shape[:2]
    idx = (bias_index[:, :, :L].long() & 0xFFFF)
    masked = idx == npos_index * 64
    pb, tb = (idx >> 6).clamp_max(wpos.shape[0] - 1), idx & 63
    w = wpos.float()[pb].permute(0, 3, 1, 2)                       # [B, H, L, L]
    if wtime is not None:
        nt = wtime.shape[0]
        wt = torch.where((tb < nt)[..., None], wtime.float()[tb.clamp_max(nt - 1)], torch.zeros((), device=w.device))
        w = w + wt.permute(0, 3, 1, 2)
    return w, masked[:, None], pb, tb


def causal_valid(pad):
    """[B, 1, L, L]: key j <= query i and j not padded (padded query rows keep their unpadded keys, as the kernels do)."""
    L = pad.shape[1]
    ii = torch.arange(L, device=pad.device)
    return (ii[None, :] <= ii[:, None])[None, None] & ~pad.bool()[:, None, None, :]


def _heads(t, H):
    B, L, D = t.shape
    return t.double().reshape(B, L, H, D // H).transpose(1, 2)


def _merge(t):
    B, H, L, dh = t.shape
    return t.transpose(1, 2).reshape(B, L, H * dh)


def attention(P, w, valid, H, zp=None, dO=None):
    """P [B, L, 4D] bf16 (U | V | Q | K), w [B, H, L, L] fp32 table sums, valid [B, 1, L, L].  -> "O" [B, L, D] with "a_O"; with zp
    and dO also "dV", "dQ", "dK" [B, L, D] (gradients w.r.t. the pre-activations) with allowances, and "dS" [B, H, L, L]."""
    B, L, D4 = P.shape
    D = D4 // 4
    dh = D // H
    _, Vc, Qc, Kc = P.split(D, -1)
    q, k, v = _heads(Qc, H), _heads(Kc, H), _heads(Vc, H)
    x = q @ k.transpose(-1, -2) + w.double()
    e_x = dh * ACC * (q.abs() @ k.abs().transpose(-1, -2)) + C * x.abs()
    sg = torch.sigmoid(x)
    zero = torch.zeros((), dtype=torch.float64, device=x.device)
    A = torch.where(valid, x * sg, zero)
    del sg
    e_A = torch.where(valid, 1.1 * e_x + SILU_SLACK * x.abs() * (1 + x.abs()), zero)
    mA = e_A + (U + L * ACC) * A.abs()                                  # per cell: A's error, its bf16 pack, the fp32 sum
    O = A @ v
    r = {"O": _merge(O), "a_O": _merge(U * O.abs() + (1 + U) * (mA @ v.abs()))}
    if dO is None:
        return r
    do = _heads(dO, H)
    dA = do @ v.transpose(-1, -2)
    e_dA = dh * ACC * (do.abs() @ v.abs().transpose(-1, -2))
    ds = dsilu(x)
    dS = torch.where(valid, dA * ds, zero)
    e_dS = torch.where(valid, ds.abs() * e_dA + dA.abs() * (0.5 * e_x + SILU_SLACK * (1 + x.abs())) + C * dS.abs(), zero)
    del x, e_x, ds, e_dA
    mS = e_dS + (U + L * ACC) * dS.abs()
    _, zV, zQ, zK = zp.split(D, -1)

    def epi(pre, a_pre, z):
        zz = _heads(z, H)
        d = dsilu(zz)
        out = pre * d
        a = d.abs() * a_pre + pre.abs() * SILU_SLACK * (1 + zz.abs()) + C * out.abs()
        return _merge(out), _merge(U * out.abs() + (1 + U) * a)

    r["dQ"], r["a_dQ"] = epi(dS @ k, mS @ k.abs(), zQ)
    r["dK"], r["a_dK"] = epi(dS.transpose(-1, -2) @ q, mS.transpose(-1, -2) @ q.abs(), zK)
    r["dV"], r["a_dV"] = epi(A.transpose(-1, -2) @ do, mA.transpose(-1, -2) @ do.abs(), zV)
    r["dS"] = dS
    return r


def table_sums(dS, valid, rows, nrows):
    """(sum of dS, sum of |dS|, cell count) per table row: rows [B, 1, L, L] the row of each cell.  -> [nrows, H], [nrows, H], [nrows]"""
    H = dS.shape[1]
    r = rows.expand_as(valid)[valid]
    ref = torch.zeros(nrows, H, dtype=torch.float64, device=dS.device)
    mass = torch.zeros_like(ref)
    for h in range(H):
        d = dS[:, h:h + 1][valid]
        ref[:, h].index_add_(0, r, d)
        mass[:, h].index_add_(0, r, d.abs())
    return ref, mass, torch.bincount(r, minlength=nrows)


# ------------------------------------------------------------------------------------------------ Adam
def f32(v):
    return float(np.float32(v))


def adam(p0, g0, m0, v0, t, lr, beta1, beta2, eps, weight_decay=0.0, grad_scale=1.0):
    """One torch.optim.Adam step (L2 weight decay, then the bias-corrected update) in fp64 from the kernel's previous p, g, m, v, at
    step t >= 1, with the fp32 values of the hyper-parameters.  -> "p", "m", "v" with allowances, "bc1", "bc2" with "a_bc1", "a_bc2"."""
    lr, b1, b2, eps, wd, gs = (f32(v) for v in (lr, beta1, beta2, eps, weight_decay, grad_scale))
    P0, G0, M0, V0 = (a.double() for a in (p0, g0, m0, v0))
    g = G0 * gs + wd * P0
    e_g = 3 * C * ((G0 * gs).abs() + (wd * P0).abs())
    m = b1 * M0 + (1 - b1) * g
    e_m = (1 - b1) * e_g + 3 * C * ((b1 * M0).abs() + ((1 - b1) * g).abs())
    v = b2 * V0 + (1 - b2) * g * g
    e_v = (1 - b2) * 2 * g.abs() * e_g + 4 * C * (b2 * V0 + (1 - b2) * g * g)
    r = {"m": m, "a_m": e_m + C * m.abs(), "v": v, "a_v": e_v + C * v}
    bc, a_bc = [], []
    for b in (b1, b2):
        bt = b ** t
        rel = math.log(2) * (LOG2_ABS * t + C * abs(t * math.log2(b))) + EXP2_REL       # __powf of the fp32 counter t
        bc.append(1 - bt)
        a_bc.append(rel * bt + C * (1 - bt))
    r.update(bc1=bc[0], a_bc1=a_bc[0], bc2=bc[1], a_bc2=a_bc[1])
    ss = lr / bc[0]
    rel_ss = a_bc[0] / bc[0] + DIV
    sq = torch.sqrt(v)
    rel_sq = DIV + 0.5 * e_v / v.clamp_min(1e-300)
    inv = 1 / math.sqrt(bc[1])
    rel_inv = RSQRT + 0.5 * a_bc[1] / bc[1]
    den = sq * inv + eps
    e_den = sq * inv * (rel_sq + rel_inv + C) + C * den
    upd = ss * (m / den)
    e_upd = ss * (e_m / den + m.abs() / den * (rel_ss + e_den / den + DIV + C))
    r["p"] = P0 - upd
    r["a_p"] = e_upd + C * r["p"].abs()
    return r


def lazy_adam_reference(p, g, m, v, rows, step, lr, betas, eps, weight_decay, grad_scale=1.0, bias_corrections=None):
    """One lazy step in fp64: FlatAdam's per-element rule (torch.optim.Adam with L2 weight decay, bias corrections of the global
    step count `step`, already ticked) on the rows `rows` of the [C, D] tensors; every other row is copied.  -> (p, m, v).
    ``bias_corrections`` = (1 - beta1^step, 1 - beta2^step) as the optimizer's state holds them, when given."""
    p, g, m, v = (t.double().clone() for t in (p, g, m, v))
    r = torch.as_tensor(sorted(set(int(i) for i in rows)), dtype=torch.long)
    b1, b2 = betas
    bc1, bc2 = bias_corrections if bias_corrections is not None else (1 - b1 ** step, 1 - b2 ** step)
    gr = g[r] * grad_scale + weight_decay * p[r]
    m[r] = b1 * m[r] + (1 - b1) * gr
    v[r] = b2 * v[r] + (1 - b2) * gr * gr
    p[r] = p[r] - lr / bc1 * (m[r] / (v[r].sqrt() / bc2 ** 0.5 + eps))
    return p, m, v
