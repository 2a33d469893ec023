"""TEST INFRASTRUCTURE - COBRA's paged pool (genrec_b200.cobra.CobraPool) restated: the page bookkeeping as plain integers, and the
paged attention (grb_cobra_paged_attention) in fp64 with the allowance of where the kernel rounds.

Pages: the free pages are a stack that starts as num_pages-1 .. 0 (page 0 goes out first).  An extend call visits its rows in order;
a row whose user gains items takes the pages its new length needs from the top of the stack, one at a time.  A release pushes the
user's pages back in reverse order, so the user's first page is on top.  Unused page-table entries are 0.

Paged attention: query r of call row b sees the keys 0 .. q_keys[r]-1 of user users[b], key j at row page_table[u, j // page_size]
page_size + j % page_size of the layer's K | V rows, then its S suffix keys.  The kernel computes q . k in fp32 (DH fused terms),
scales it, keeps a running max and sum with __expf in fp32 over fixed 128-key ranges merged in order, divides, and rounds the output
to bf16 once.  Allowance per output element: half a bf16 ulp of the result (U |o|), plus, on sum_j p_j |v_j|, the fp32 error of the
scores (DH + 2 roundings of each product magnitude, times the scale), of __expf's argument (|s - max| C) and of ex2.approx (2^-21),
and C per term of the fp32 sums.
"""
from __future__ import annotations

import math

import torch

from tests.attention_reference import U

C32 = 2.0 ** -24


class PageModel:
    """the page bookkeeping of CobraPool as plain integers"""

    def __init__(self, max_users, num_pages, page_size, C, max_items):
        self.page_size, self.C, self.max_items = page_size, C, max_items
        self.lengths = [0] * max_users
        self.pages = [[] for _ in range(max_users)]
        self.free = list(range(num_pages - 1, -1, -1))
        self.cols = -(-max_items * (C + 1) // page_size)

    def _need(self, items):
        return -(-items * (self.C + 1) // self.page_size)

    def fits(self, users, counts):
        """whether an extend of counts[b] items for users[b] stays within max_items and the free pages"""
        if any(self.lengths[u] + k > self.max_items for u, k in zip(users, counts)):
            return False
        return sum(self._need(self.lengths[u] + k) - self._need(self.lengths[u]) for u, k in zip(users, counts)) <= len(self.free)

    def extend(self, users, counts):
        assert self.fits(users, counts)
        for u, k in zip(users, counts):
            if k:
                while len(self.pages[u]) < self._need(self.lengths[u] + k):
                    self.pages[u].append(self.free.pop())
                self.lengths[u] += k

    def release(self, users):
        for u in users:
            self.free.extend(reversed(self.pages[u]))
            self.pages[u] = []
            self.lengths[u] = 0

    def table(self):
        t = torch.zeros(len(self.pages), self.cols, dtype=torch.int32)
        for u, p in enumerate(self.pages):
            t[u, :len(p)] = torch.tensor(p, dtype=torch.int32)
        return t

    def rows(self, u, n):
        """the K | V row indices of user u's positions 0 .. n-1"""
        return [self.pages[u][j // self.page_size] * self.page_size + j % self.page_size for j in range(n)]


def key_rows(page_table, page_size, u, n):
    return [int(page_table[u, j // page_size]) * page_size + j % page_size for j in range(n)]


def paged_attention(q, k, v, page_table, page_size, users, q_off, q_keys, H, suf=None, anc=None, S=0):
    """fp64 of grb_cobra_paged_attention on the kernel's bf16 operands (CPU tensors).  q [R, D]; k / v [rows, D] (the layer's K and V
    rows); page_table None: user b's key j is row b page_size + j.  suf [steps, R, 3D], anc [R, S-1].  -> (out [R, D] fp64, allowance
    [R, D] fp64)"""
    R, D = q.shape
    dh = D // H
    scale = 1.0 / math.sqrt(dh)
    out = torch.empty(R, D, dtype=torch.float64)
    allow = torch.empty(R, D, dtype=torch.float64)
    for b in range(len(q_off) - 1):
        u = int(users[b]) if users is not None else b
        for r in range(int(q_off[b]), int(q_off[b + 1])):
            n = int(q_keys[r])
            rows = key_rows(page_table, page_size, u, n) if page_table is not None else [u * page_size + j for j in range(n)]
            ks, vs = [k[rows].double()], [v[rows].double()]
            for s in range(S):
                row = int(anc[r, s]) if s < S - 1 else r
                ks.append(suf[s, row, D:2 * D].double()[None])
                vs.append(suf[s, row, 2 * D:].double()[None])
            kk, vv = torch.cat(ks).view(-1, H, dh), torch.cat(vs).view(-1, H, dh)
            qq = q[r].double().view(H, dh)
            prod = torch.einsum("hd,jhd->hjd", qq, kk)
            sc = prod.sum(-1) * scale
            p = torch.softmax(sc, dim=-1)
            o = torch.einsum("hj,jhd->hd", p, vv)
            mag = prod.abs().sum(-1).max(-1).values * scale                       # [H]
            smax = sc.abs().max(-1).values
            e = 2.0 ** -21 + C32 * ((dh + 2) * mag + 2 * smax + kk.shape[0] + 8)
            out[r] = o.reshape(-1)
            allow[r] = (U * o.abs() + e[:, None] * torch.einsum("hj,jhd->hd", p, vv.abs())).reshape(-1)
    return out, allow


def dense_softmax(q, keys, values, H):
    """softmax(q k^T / sqrt(dh)) v per head on explicit key lists: q [D], keys / values [n, D] -> [D] fp64"""
    D = q.shape[0]
    dh = D // H
    qq, kk, vv = q.double().view(H, dh), keys.double().view(-1, H, dh), values.double().view(-1, H, dh)
    p = torch.softmax(torch.einsum("hd,jhd->hj", qq, kk) / math.sqrt(dh), dim=-1)
    return torch.einsum("hj,jhd->hd", p, vv).reshape(-1)
