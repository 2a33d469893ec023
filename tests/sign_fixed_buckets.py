"""The sign-fixed relative-position bias for the oracle: bucket(i - j) for cell (i, j), a non-uniform table on the causal
triangle, where the reference evaluates bucket(j - i) and lands every causal cell in bucket 0 (SURVEY.md section 0).
Tests swap it in for ``oracle.hstu.position_bias`` with pytest's ``monkeypatch``."""
import torch
import torch.nn.functional as F


def sign_fixed_position_bias(table: torch.Tensor, L: int, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    from oracle import hstu as oh
    pos = torch.arange(L, device=table.device)
    rel = pos.unsqueeze(1) - pos.unsqueeze(0)                    # [i, j] = i - j
    return F.embedding(oh.position_bucket(rel, num_buckets, max_distance), table).permute(2, 0, 1)


def use_sign_fixed_oracle(monkeypatch) -> None:
    from oracle import hstu as oh
    monkeypatch.setattr(oh, "position_bias", sign_fixed_position_bias)
