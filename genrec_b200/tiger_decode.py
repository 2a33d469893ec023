"""Device-side trie-constrained beam search for TIGER (SURVEY.md section 8 row f4).

Drop-in for the decode loop of ``genrec/models/tiger.py:312-452`` (``Tiger.generate``): the encoder / decoder forward stays whatever
module the caller owns (``model._encode_context`` / ``model._decode_step``, the reference's own methods); the per-step post-processing -
legal-token mask from the trie, temperature softmax, candidate ranking, duplicate removal, trie descent - is two launches of
``libgenrec_b200`` (csrc/beam.cuh) instead of Python loops over batch x beam with ``.item()`` calls.

    trie = TrieCSR.build(valid_item_ids).to(device)          # once          (build_trie, tiger.py:49-69)
    out = generate(model, user_ids, item_ids, token_types, seq_mask, temperature=0.2, n_top_k_candidates=10, trie=trie)

Candidate sampling is ``torch.multinomial`` on the probabilities the kernel produced, as in the reference (tiger.py:385-386): with
the same generator state and the same logits the same candidates are drawn.
"""
from __future__ import annotations

from typing import NamedTuple, Optional

import torch

from ._lib import call, ptr, require_cuda, workspace


class TigerGenerationOutput(NamedTuple):      # (tiger.py:78-83)
    sem_ids: torch.Tensor
    log_probas: torch.Tensor


class TrieCSR:
    """The reference's dict trie (tiger.py:40-69) as three int32 arrays.  Node 0 is the root; the nodes of level l are the distinct
    prefixes of length l + 1 in lexicographic order, so the children of a node are contiguous and sorted by token."""

    def __init__(self, child_off: torch.Tensor, child_tok: torch.Tensor, child_node: torch.Tensor, depth: int, leaf_row: torch.Tensor):
        self.child_off, self.child_tok, self.child_node, self.depth = child_off, child_tok, child_node, depth
        self.leaf_row = leaf_row      # [n_nodes] int64: the smallest row of valid_item_ids holding a leaf's tuple, -1 for other nodes

    @property
    def n_nodes(self) -> int:
        return self.child_off.numel() - 1

    @staticmethod
    def build(valid_item_ids: torch.Tensor) -> "TrieCSR":
        v = valid_item_ids
        if v.dim() == 3:
            v = v.reshape(-1, v.size(-1))
        elif v.dim() == 1:
            v = v.unsqueeze(0)
        v = v.detach().to("cpu", torch.int64)
        n, depth = v.shape
        parents, toks = [], []
        base_prev, inv_prev = 0, torch.zeros(n, dtype=torch.int64)          # level -1: everything hangs off the root
        base, rep = 1, torch.zeros(0, dtype=torch.int64)
        for lvl in range(depth):
            uniq, inv = torch.unique(v[:, :lvl + 1], dim=0, return_inverse=True)
            rep = torch.full((uniq.size(0),), n, dtype=torch.int64).scatter_reduce_(0, inv, torch.arange(n), "amin")   # a row per node
            parents.append((base_prev + inv_prev[rep]) if lvl > 0 else torch.zeros(uniq.size(0), dtype=torch.int64))
            toks.append(uniq[:, lvl])
            base_prev, inv_prev = base, inv
            base += uniq.size(0)
        n_nodes = base
        leaf_row = torch.full((n_nodes,), -1, dtype=torch.int64)
        leaf_row[n_nodes - rep.numel():] = rep                             # the last level's nodes are the leaves
        parent = torch.cat(parents) if parents else torch.zeros(0, dtype=torch.int64)
        tok = torch.cat(toks) if toks else torch.zeros(0, dtype=torch.int64)
        child = torch.arange(1, n_nodes, dtype=torch.int64)
        # nodes were numbered level by level in lexicographic order, so edges are already grouped by parent with ascending tokens
        counts = torch.bincount(parent, minlength=n_nodes)
        off = torch.zeros(n_nodes + 1, dtype=torch.int64)
        off[1:] = torch.cumsum(counts, 0)
        order = torch.argsort(parent * (int(tok.max().item()) + 1 if tok.numel() else 1) + tok, stable=True)
        return TrieCSR(off.to(torch.int32), tok[order].to(torch.int32), child[order].to(torch.int32), depth, leaf_row)

    def to(self, device) -> "TrieCSR":
        return TrieCSR(self.child_off.to(device), self.child_tok.to(device), self.child_node.to(device), self.depth,
                       self.leaf_row.to(device))

    def rows(self, nodes: torch.Tensor) -> torch.Tensor:
        """Catalog row of the leaf each node id stands for (int64), -1 for dead (-1) and non-leaf nodes."""
        return torch.where(nodes >= 0, self.leaf_row[nodes.long().clamp(min=0)], -1)


def trie_log_softmax(logits: torch.Tensor, nodes: Optional[torch.Tensor], trie: Optional[TrieCSR], vocab_offset: int, num_embeddings: int,
                     temperature: float):
    """logits [R, V] fp32 -> (probs, log_probs) of ``masked_fill(~legal, -1e32) / temperature`` (tiger.py:364-384)."""
    require_cuda(logits)
    x = logits.detach().float().contiguous()
    R, V = x.shape
    probs, logp = torch.empty_like(x), torch.empty_like(x)
    use = trie is not None
    if use:
        nodes = nodes.to(torch.int32).contiguous()
    call(x.device, "grb_trie_log_softmax", ptr(x), R, V, ptr(nodes) if use else None, ptr(trie.child_off) if use else None,
         ptr(trie.child_tok) if use else None, trie.n_nodes if use else 0, 1 if use else 0, int(vocab_offset), int(num_embeddings),
         float(temperature), ptr(probs), ptr(logp))
    return probs, logp


MAX_BEAMS = 1024                   # K: beams per user
MAX_CANDIDATES = 262144            # K * KK: candidates per user and step


def candidates_per_beam(K: int, num_item_embeddings: int) -> int:
    return min(K * 6, num_item_embeddings)                                       # (tiger.py:349-350)


def check_width(K: int, KK: int) -> None:
    """Refuse a beam step the kernels cannot run, before anything is launched."""
    if not 1 <= K <= MAX_BEAMS:
        raise ValueError(f"n_top_k_candidates = {K} is outside 1 .. {MAX_BEAMS} (beams per user)")
    if KK < 1 or K * KK > MAX_CANDIDATES:
        raise ValueError(f"K * KK = {K} * {KK} = {K * KK} candidates per user and step; the limit is {MAX_CANDIDATES} "
                         f"(KK = min(6 K, num_item_embeddings))")


def beam_select(beam_seqs: torch.Tensor, beam_logps: torch.Tensor, cand_tok: torch.Tensor, cand_logp: torch.Tensor,
                nodes: Optional[torch.Tensor], trie: Optional[TrieCSR]):
    """One beam update (tiger.py:386-441): beam_seqs [B, K, S] int64, beam_logps [B, K], cand_tok / cand_logp [B, K, KK] ->
    (new_seqs [B, K, S+1], new_logps [B, K], new_nodes [B, K] int32 | None)."""
    B, K, KK = cand_tok.shape
    check_width(K, KK)
    require_cuda(beam_logps, cand_tok, cand_logp)
    S = beam_seqs.size(2)
    dev = beam_logps.device
    seqs = beam_seqs.to(torch.int64).contiguous()
    new_seqs = torch.empty(B, K, S + 1, dtype=torch.int64, device=dev)
    new_logps = torch.empty(B, K, dtype=torch.float32, device=dev)
    use = trie is not None
    new_nodes = torch.empty(B, K, dtype=torch.int32, device=dev) if use else None
    nodes_c = nodes.to(torch.int32).contiguous() if use else None
    args = (ptr(seqs) if S > 0 else None, ptr(beam_logps.float().contiguous()), ptr(cand_tok.to(torch.int64).contiguous()),
            ptr(cand_logp.float().contiguous()), ptr(nodes_c), ptr(trie.child_off) if use else None, ptr(trie.child_tok) if use else None,
            ptr(trie.child_node) if use else None, trie.n_nodes if use else 0, B, K, KK, S, ptr(new_seqs), ptr(new_logps), ptr(new_nodes))
    if K <= 32 and K * KK <= 1024:                                           # one CTA sorts a row's candidates
        call(dev, "grb_beam_select", *args)
    else:
        ws = workspace(dev, "grb_beam_select_wide_workspace_bytes", B, K, KK)
        call(dev, "grb_beam_select_wide", *args, ptr(ws))
    return new_seqs, new_logps, new_nodes


@torch.no_grad()
def beam_search(decode_step, B: int, K: int, sem_id_dim: int, num_item_embeddings: int, device, temperature: float = 0.2,
                trie: Optional[TrieCSR] = None, generator: Optional[torch.Generator] = None, draws=None, return_nodes: bool = False):
    """The loop of Tiger.generate (tiger.py:352-452).  ``decode_step(beam_seqs [B*K, S] int64) -> logits [B*K, V]`` is the caller's
    decoder; ``draws`` (test hook) replaces torch.multinomial by recorded candidate indices, one [B*K, KK] tensor per step.
    ``return_nodes``: also return the trie node each final beam reached ([B, K] int32, None without a trie)."""
    KK = candidates_per_beam(K, num_item_embeddings)
    check_width(K, KK)
    beam_seqs = torch.empty(B, K, 0, dtype=torch.long, device=device)
    beam_logps = torch.zeros(B, K, device=device)
    nodes = torch.zeros(B, K, dtype=torch.int32, device=device) if trie is not None else None
    for step in range(sem_id_dim):
        logits = decode_step(beam_seqs.view(B * K, -1))
        vocab_offset = step * num_item_embeddings
        probs, logp = trie_log_softmax(logits, nodes.view(-1) if nodes is not None else None, trie, vocab_offset, num_item_embeddings,
                                       temperature)
        cand = draws[step].to(device) if draws is not None else torch.multinomial(probs, num_samples=KK, generator=generator)
        cand_logp = torch.gather(logp, 1, cand)
        beam_seqs, beam_logps, nodes = beam_select(beam_seqs, beam_logps, (cand - vocab_offset).view(B, K, KK), cand_logp.view(B, K, KK),
                                                   nodes, trie)
    out = TigerGenerationOutput(sem_ids=beam_seqs, log_probas=beam_logps)
    return (out, nodes) if return_nodes else out


@torch.no_grad()
def generate(model, user_input_ids: torch.Tensor, item_input_ids: torch.Tensor, token_type_ids: torch.Tensor,
             seq_mask: Optional[torch.Tensor] = None, temperature: float = 0.2, n_top_k_candidates: int = 10,
             valid_item_ids: Optional[torch.Tensor] = None, use_trie: bool = True, trie: Optional[TrieCSR] = None,
             generator: Optional[torch.Generator] = None) -> TigerGenerationOutput:
    """Same arguments and result as ``Tiger.generate`` (tiger.py:312-323) for any module with the reference's ``_encode_context`` /
    ``_decode_step`` / ``sem_id_dim`` / ``num_item_embeddings``; ``trie`` (a TrieCSR already on the device) avoids rebuilding it."""
    B, K = user_input_ids.size(0), n_top_k_candidates
    check_width(K, candidates_per_beam(K, model.num_item_embeddings))
    device = user_input_ids.device
    memory, memory_mask = model._encode_context(user_input_ids, item_input_ids, token_type_ids, seq_mask)
    memory = memory.unsqueeze(1).expand(-1, K, -1, -1).reshape(B * K, memory.size(1), -1)
    memory_mask = memory_mask.unsqueeze(1).expand(-1, K, -1).reshape(B * K, -1)
    if use_trie and trie is None:
        trie = getattr(model, "_grb_trie", None)
        if trie is None:
            trie = TrieCSR.build(valid_item_ids).to(device)
            model._grb_trie = trie
    if not use_trie:
        trie = None

    def decode_step(tgt):
        if tgt.numel() == 0:
            return model._decode_step(memory, memory_mask, None, None)
        types = torch.arange(tgt.size(1), device=device).unsqueeze(0).expand(tgt.size(0), -1)
        return model._decode_step(memory, memory_mask, tgt, types)

    return beam_search(decode_step, B, K, model.sem_id_dim, model.num_item_embeddings, device, temperature, trie, generator)
