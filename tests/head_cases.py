"""TEST INFRASTRUCTURE - the cross-entropy head cases the GPU tests share: seeded head operands and the logits-path selection the
top-k, candidates and rank heads are checked against, and the head-loss C ABI call with its fp64 reference."""
import torch

from tests.head_reference import reference
EPS = 1e-5
NEG = float("-inf")


def _dev():
    return torch.device("cuda:0")


def _to_dev(case):
    from genrec_b200 import functional as Fn
    c = {k: (v.to(_dev()).contiguous() if v is not None else None) for k, v in case.items()}
    c["tb"] = Fn.cast_bf16(c["table"])
    return c


def _select(logits, k, exclude=None):
    logits = logits.clone()
    C = logits.shape[1]
    logits[:, 0] = NEG
    if exclude is not None and exclude.shape[1]:
        logits.scatter_(1, torch.where((exclude >= 1) & (exclude < C), exclude, 0), NEG)
    if C < k:                                   # fewer items than slots: the rest is (-inf, 0)
        logits = torch.cat([logits, logits.new_full((logits.shape[0], k - C), NEG)], 1)
    s, i = torch.sort(logits, dim=1, descending=True, stable=True)
    s, i = s[:, :k], i[:, :k]
    return s, torch.where(s == NEG, torch.zeros_like(i), i)


def _assert_same(got, ref):
    s, i = got
    rs, ri = ref
    assert torch.equal(s, rs), (s - rs).abs().max()
    assert torch.equal(i, ri), (i != ri).nonzero()[:8]


def _head(R, D, C, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R, D, generator=g).cuda()
    ln_g = (1 + 0.1 * torch.randn(D, generator=g)).cuda()
    ln_b = (0.1 * torch.randn(D, generator=g)).cuda()
    tb = (0.05 * torch.randn(C, D, generator=g)).to(torch.bfloat16).cuda()
    return x, ln_g, ln_b, tb


def _call(c, *, dx=None, dtable=None, dg=None, db=None, ws=None, loss_only=False, tg=None):
    """grb_head_loss_forward_backward through the C ABI; zeroed gradient buffers and workspace unless given."""
    from genrec_b200 import _lib
    from genrec_b200._lib import check, ptr, stream_ptr
    lib = _lib.load()
    x, tb = c["x"], c["tb"]
    T, D = x.shape
    C = tb.shape[0]
    dev = x.device
    if ws is None:
        ws = torch.zeros(lib.grb_head_workspace_bytes(T, D, C), dtype=torch.uint8, device=dev)
    if not loss_only:
        dx = torch.empty_like(x) if dx is None else dx
        dtable = torch.zeros(C, D, device=dev) if dtable is None else dtable
        dg = torch.zeros(D, device=dev) if dg is None else dg
        db = torch.zeros(D, device=dev) if db is None else db
    loss = torch.empty((), dtype=torch.float32, device=dev)
    check(lib.grb_head_loss_forward_backward(ptr(x), ptr(c["ln_g"]), ptr(c["ln_b"]), EPS, ptr(tb), ptr(c["tg"] if tg is None else tg), T, D, C,
                                             ptr(loss), ptr(dx), ptr(dtable), ptr(dg), ptr(db), ptr(ws), stream_ptr(dev)))
    torch.cuda.synchronize()
    return {"loss": loss.item(), "dx": dx, "dg": dg, "db": db, "dE": dtable}


def _reference(c, chunk=2048):
    from genrec_b200 import functional as Fn
    xf, _, st = Fn.layernorm_fwd(c["x"], c["ln_g"], c["ln_b"], EPS)     # ln_fwd_kernel, as the head launches it: the same bits
    return reference(c["x"], st, xf, c["ln_g"], c["tb"], c["tg"], chunk=chunk)
