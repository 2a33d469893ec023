"""TEST INFRASTRUCTURE - the harness the fp64 check modules (tests/test_*_exact_gpu.py) share: a per-module ledger of the worst
error / allowance of every checked quantity with the fixture that prints it, a spy on the functional calls of a backward, the
dropout shim and the packed T5 core reference of the TIGER and COBRA steps, the bf16-autocast yardstick of the whole-model checks,
and the small seeded inputs."""
import pytest
import torch

from tests import attention_reference as ar
from tests import dense_reference as dr
from tests import tiger_reference as tr

DEV = torch.device("cuda:0")
# fp32 flush-to-zero (--use_fast_math) of products and partial sums below 2^-126, over up to 2^26 terms: padded keys carry values
# of 1e-37 into the K | V gradient GEMMs
FTZ = 2.0 ** -100


class Ledger:
    """One module's worst error / allowance per quantity and the case where it occurred.  `fixture()` makes the module-scoped autouse
    fixture that prints them under `title` when the module ends (pytest -s); bind it as a module attribute.  `floor` is added to
    every allowance `check` is given."""

    def __init__(self, title, width=12, floor=0.0):
        self.title, self.width, self.floor, self.worst = title, width, floor, {}

    def fixture(self):
        @pytest.fixture(scope="module", autouse=True)
        def _error_table():
            yield
            if self.worst:
                print("\n" + self.title)
                for name, (w, case) in sorted(self.worst.items()):
                    print(f"  {name:{self.width}s} {w:8.4f}   {case}")
        return _error_table

    def record(self, case, name, w, tol=dr.TOL):
        if name not in self.worst or w > self.worst[name][0]:
            self.worst[name] = (w, case)
        return None if w <= tol else f"{name} {w:.3g}"

    def check(self, case, items):
        """items: (name, got, ref, allowance).  Records each worst ratio and fails on any above dense_reference.TOL."""
        bad = [self.record(case, n, dr.worst(g, r, a + self.floor if self.floor else a)) for n, g, r, a in items]
        bad = [b for b in bad if b]
        assert not bad, (case, bad)

    def check_core(self, case, err, kind):
        """err: attention_reference.errors of one attention core; kind: its attention_reference tolerance set"""
        for n, (w, f) in err.items():
            tw, tf = ar.tolerance(kind, n)
            self.record(case, "core " + n, w / tw, 1.0)
            self.record(case, "core " + n + " frob", f / tf, 1.0)
        bad = ar.violations(err, kind)
        assert not bad, (case, bad)


class Spy:
    """records the outputs of the functional calls made while it is active, by name, in call order.  wraps: {module: names}"""

    def __init__(self, monkeypatch, wraps):
        self.calls = []
        for mod, names in wraps.items():
            for n in names:
                monkeypatch.setattr(mod, n, self._wrap(n, getattr(mod, n)))

    def _wrap(self, name, fn):
        def spy(*a, **k):
            out = fn(*a, **k)
            self.calls.append((name, out))
            return out
        return spy

    def take(self, *names):
        assert [n for n, _ in self.calls] == list(names), [n for n, _ in self.calls]
        got = [out for _, out in self.calls]
        self.calls.clear()
        return got


def _dy(shape, seed):
    """small integers / 64: every masked bf16 cast of it is exact"""
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(-64, 65, shape, generator=g).float() / 64).to(DEV)


def _seeded(shape, seed, scale=1.0, shift=0.0):
    return (scale * torch.randn(shape, generator=torch.Generator().manual_seed(seed)) + shift).to(DEV)


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _cid(c):
    return "-".join(str(v) for v in c)


def row_pass():
    """rows one pass of the gate kernels' grid covers: row_grid caps at 8 CTAs per SM, of 8 rows each"""
    return 8 * _sms() * 8


def _packed_core_ref(Q, K, V, A, dAb, H, bias, offs, Lq, scale, p, seed, site):
    """the fp64 core per sequence with the packed keys (as test_tiger_jagged_gpu._core_check) -> (ref, rows of Q / of K per seq)"""
    from genrec_b200 import t5_attention as t5
    mx = max(b - a for a, b in zip(offs, offs[1:]))
    B = len(offs) - 1
    mask = (tr.attn_mask_packed_self(Q.shape[0], H, mx, p, seed, site, DEV) if Lq == 0
            else tr.attn_mask_packed_cross(B, H, Lq, mx, p, seed, site, DEV))
    names = ("out", "dq", "dk", "dv")
    ref = {k: [] for n in names for k in (n, "a_" + n)}
    db = adb = None
    saved = ar.attn_keep
    try:
        for b in range(B):
            r0, r1 = offs[b], offs[b + 1]
            n = r1 - r0
            if Lq == 0:
                keep = mask[r0:r1, :, :n].transpose(0, 1)[None]
                q, o, do = Q[r0:r1][None], A[r0:r1][None], dAb[r0:r1][None]
                bk = t5.relative_position_buckets(n, n).to(DEV)
            else:
                keep = mask[b:b + 1, :, :, :n]
                q, o, do = Q[b:b + 1], A[b:b + 1], dAb[b:b + 1]
                bk = None
            ar.attn_keep = lambda *a, **k: keep
            r = ar.t5_reference(q, K[r0:r1][None], V[r0:r1][None], H, bias, bk, None, False, scale, do, o, p, seed, site)
            for nm in names:
                ref[nm].append(r[nm][0])
                ref["a_" + nm].append(r["a_" + nm][0])
            if bias is not None:
                db = r["dbias"] if db is None else db + r["dbias"]
                adb = r["a_dbias"] if adb is None else adb + r["a_dbias"]
    finally:
        ar.attn_keep = saved
    ref = {k: torch.cat(v) for k, v in ref.items()}
    if bias is not None:
        ref["dbias"], ref["a_dbias"] = db, adb
    return ref


class _TorchDropout:
    """genrec_b200.tiger's F: dropout draws a keep-scale mask, records it and applies it; everything else is torch.nn.functional"""

    def __init__(self):
        self.masks = []

    def dropout(self, x, p=0.5, training=True):
        if not training or p == 0:
            return x
        m = torch.where(torch.rand(x.shape, device=x.device) >= p, ar.keep_scale(p)[1], 0.0)
        self.masks.append(m.double())
        return x * m

    def __getattr__(self, name):
        return getattr(torch.nn.functional, name)


def autocast_yardstick(rows, small):
    """rows: (name, ours Frobenius, reference-autocast Frobenius, ours max-norm, reference-autocast max-norm) relative errors against
    the fp32 oracle; small: the names of tensors of < 4096 elements.  Prints the table (pytest -s) and asserts the yardstick."""
    lines = ["| tensor | ours, Frobenius | reference autocast, Frobenius | ratio | ours, max-norm | reference autocast, max-norm | ratio |",
             "|---|---|---|---|---|---|---|"]
    lines += [f"| {n} | {a:.2e} | {b:.2e} | {a / max(b, 1e-12):.2f} | {c:.2e} | {d:.2e} | {c / max(d, 1e-12):.2f} |" for n, a, b, c, d in rows]
    print("\n".join(lines))
    # Yardstick.  Both columns are one realisation of bf16 rounding noise, so the ratio of the two scatters from tensor to tensor
    # (and, for ours, from build to build: +-10 % on the matrices, a factor ~2 on a 399-entry bias table whose every entry is a
    # cancelling sum of ~10^5 noisy terms).
    #   weight matrices / embedding table / dX (>= 4096 elements): Frobenius error <= 1.1 x the reference algorithm's own
    #       bf16-autocast error, and the geometric mean of the ratio over all of them <= 1.0;
    #   vectors of < 4096 elements (bias tables, norm parameters): <= 3 x each, geometric mean <= 1.25;
    #   the max-norm (one worst element out of up to 1.5 M) is reported and held within 3 x.
    import math
    big_r = [a / b for n, a, b, c, d in rows if n not in small and n != "loss" and b > 0]
    small_r = [a / b for n, a, b, c, d in rows if n in small and b > 0]
    gm = lambda v: math.exp(sum(math.log(max(x, 1e-6)) for x in v) / max(len(v), 1))
    print(f"geometric mean of ours / reference-autocast: matrices {gm(big_r):.3f} ({len(big_r)}), small vectors {gm(small_r):.3f} ({len(small_r)})")
    bad = [(n, a, b, c, d) for n, a, b, c, d in rows if a > (3.0 if n in small else 1.1) * b + 5e-4 or c > 3.0 * d + 1e-3]
    assert not bad, bad
    assert gm(big_r) <= 1.0 and gm(small_r) <= 1.25, (gm(big_r), gm(small_r))
