import torch


def relerr(a: torch.Tensor, ref: torch.Tensor) -> float:
    """max-norm relative error: |a - ref|_inf / |ref|_inf (the reference's autocast semantics: SURVEY.md Appendix B)."""
    a, ref = a.detach().float().cpu(), ref.detach().float().cpu()
    d = ref.abs().max().item()
    return ((a - ref).abs().max().item() / d) if d > 0 else (a - ref).abs().max().item()


def budget(golden_ac: torch.Tensor, golden: torch.Tensor, slack: float = 1.5, floor: float = 4e-3) -> float:
    """bf16 tolerance = slack x the reference's OWN bf16-autocast error on this tensor (+ a small floor)."""
    return slack * relerr(golden_ac, golden) + floor


HSTU_LAYER_KEYS = {
    "projection.weight": "proj_w", "projection.bias": "proj_b",
}


def make_batch(B, L, V, seed, pad=True, device="cpu"):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, V + 1, (B, L), generator=g)
    gaps = torch.randint(1, 3 * 86400, (B, L), generator=g)
    gaps[:, ::5] = torch.randint(1, 50, (B, (L + 4) // 5), generator=g)
    ts = 1_300_000_000 + torch.cumsum(gaps, 1)
    tg = torch.roll(ids, -1, 1)
    tg[:, -1] = torch.randint(1, V + 1, (B,), generator=g)
    if pad and B >= 3 and L >= 3:
        n1 = max(1, L // 3)
        ids[1, :n1] = 0; ts[1, :n1] = 0; tg[1, : n1 - 1] = 0
        ids[2, :] = 0; ts[2, :] = 0; tg[2, :] = 0
        tg[2, -1] = 7
    return ids.to(device), ts.to(device), tg.to(device)


def close(a: torch.Tensor, ref: torch.Tensor, rel: float, floor: float = 1e-4) -> bool:
    """|a - ref|_inf <= rel * max(|ref|_inf, floor)  (floor: gradients that are analytically zero, e.g. the key-projection
    bias under a softmax, are pure rounding noise in both implementations)."""
    a, ref = a.detach().float().cpu(), ref.detach().float().cpu()
    return (a - ref).abs().max().item() <= rel * max(ref.abs().max().item(), floor)


def frob_relerr(a: torch.Tensor, ref: torch.Tensor) -> float:
    a, ref = a.detach().double().cpu(), ref.detach().double().cpu()
    d = ref.norm().item()
    return (a - ref).norm().item() / d if d > 0 else (a - ref).norm().item()
