// genrec_b200 - rank of each row's target item under the tied-embedding head without the [R, C] logits (grb_head_rank).
//
//   rank[r] = 1 + #{ j in 1..C-1, j not excluded : s_j > s_t  or  (s_j == s_t and j < t) },   s = LN(x[r]) . E^T,  t = targets[r]
//
// the rule eval_rank_kernel (rowwise.cuh) applies to stored logits.  Rows whose target is 0, out of 1..C-1 or in the row's
// exclusion list are not ranked (rank 0).  Launches after the LayerNorm and the exclusion sort (head_sweep.cuh):
//   head_rank_gather_kernel    one warp per row: the target's bf16 table row -> G [R, D]; which rows are ranked; counts = 0
//   head_rank_target_kernel    one CTA per row tile: the sweep's steps on one tile, row tile mt of LN(x) against tile mt of G,
//                              keeping the diagonal.  The same A row, the same B column and the same tc_mainloop give the fp32
//                              bits the sweep computes for column t, so the target never counts itself and ties are ordered
//                              exactly.
//   head_rank_kernel           TMA + mbarrier + wgmma (tc_mainloop with A resident, K = D), one CTA per (row tile, item range)
//                              as sweep_range (head_sweep.cuh) assigns them.  tc_mainloop is the wgmma sequence grb_head_logits
//                              runs, so every score has the bits of its logit.  Each consumer thread compares its 64
//                              accumulators straight from the registers against the target scores of its two rows; at the end
//                              of the range 4 lanes per row add up and one atomicAdd per (row, CTA) adds the range's count.
//                              Integer sums: the result does not depend on the split.
//   head_rank_finish_kernel    rank = 1 + count -> ranks; Recall / NDCG @{1,5,10} with rank_metrics_add, as eval_rank_kernel
#pragma once
#include "head_sweep.cuh"
#include "rowwise.cuh"

namespace grb {

struct HeadRankArgs {
    int R, C, E;
    int splits, num_n, kblocks;
    const long long* targets;   // [R]
    const int* excl;            // [R, E] sorted int32 (INT_MAX = ignored entry), or null
    int* tid;                   // [R] the target when the row is ranked, else 0
    float* tscore;              // [R] the target's score
    int* cnt;                   // [R] items ranked above the target
    float* metrics;             // [6] accumulated, or null
    int* ranks;                 // [R], or null
};

// ------------------------------------------------------------------------------------------------ target rows
__global__ void __launch_bounds__(256) head_rank_gather_kernel(const bf16* __restrict__ table, int D, HeadRankArgs a, bf16* __restrict__ G) {
    pdl_wait();
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= a.R) return;
    const long long t = a.targets[r];
    bool ok = t >= 1 && t < a.C;
    if (ok && a.excl) ok = !sweep_excluded(a.excl + (size_t)r * a.E, a.E, (int)t);
    const uint4* src = reinterpret_cast<const uint4*>(table + (size_t)(ok ? t : 0) * D);
    uint4* dst = reinterpret_cast<uint4*>(G + (size_t)r * D);
    for (int c = lane; c < D / 8; c += 32) dst[c] = ok ? src[c] : make_uint4(0u, 0u, 0u, 0u);
    if (lane == 0) {
        a.tid[r] = ok ? (int)t : 0;
        a.cnt[r] = 0;
    }
}

// ------------------------------------------------------------------------------------------------ target scores
__global__ void __launch_bounds__(TC_THREADS, 1)
    head_rank_target_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmG, HeadRankArgs a) {
    extern __shared__ unsigned char rank_smem_raw[];
    const RankSmem s = rank_cta_init(rank_smem_raw, &tmA, &tmG);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int m0 = blockIdx.x * TC_BM;
    if (warp < 4) {
        if (warp == 0 && lane == 0) rank_produce(&tmA, &tmG, s, m0, m0, 1, a.kblocks);
        return;
    }
    const int g = (warp >> 2) - 1;
    int stage = 0;
    uint32_t phase = 0;
    float acc[64];
    mbar_wait(s.a_bar, 0);
    tc_mainloop<0, 0, RANK_STAGES, true>(acc, s.sA, s.sB, s.full_bar, s.empty_bar, 0, a.kblocks, g, stage, phase);
    // tile row rr meets G column rr.  The thread holds columns 8 j + 2 (lane % 4) + e and rr % 8 = lane / 4, so the diagonal lies
    // with the lanes where lane % 4 = lane / 8, at e = (lane / 4) % 2 and j = rr / 8.
    if ((lane & 3) != (lane >> 3)) return;
    const int e = (lane >> 2) & 1;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int rr = rank_frag_row(g, i), jj = rr >> 3;
        float v = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) v = j == jj ? (e ? acc[4 * j + 2 * i + 1] : acc[4 * j + 2 * i]) : v;
        if (m0 + rr < a.R) a.tscore[m0 + rr] = v;
    }
}

// ------------------------------------------------------------------------------------------------ the sweep
// Adds to cnt[i] the columns of one 128-item tile (first id n0) that rank above the target of accumulator row i.  Column k = 8 j + e
// of this thread is item n0 + cb + k.  EDGE: the tile holds item 0 or ids >= C (TMA zero-fill), which never count.
template <bool EDGE, bool EXCL>
GRB_DEVINL void rank_count_tile(const float (&acc)[64], const float (&st)[2], const int (&tgt)[2], const int* const (&ex)[2], int E, int n0,
                                int cb, int C, int (&cnt)[2]) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int tl = tgt[i] - n0 - cb;          // a tie counts when k < tl (a lower id); tgt = 0 (row not ranked) never counts
        const int lo = (n0 == 0 ? 1 : 0) - cb, hi = C - n0 - cb;
        int c = 0;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int k = 8 * j + e;
                const float v = acc[4 * j + 2 * i + e];
                bool h = v > st[i] || (v == st[i] && k < tl);
                if (EDGE) h = h && k >= lo && k < hi;
                if (EXCL && h) h = !sweep_excluded(ex[i], E, n0 + cb + k);
                c += h;
            }
        }
        cnt[i] += c;
    }
}

template <bool EXCL>
__global__ void __launch_bounds__(TC_THREADS, 1)
    head_rank_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, HeadRankArgs a) {
    extern __shared__ unsigned char rank_smem_raw[];
    const RankSmem s = rank_cta_init(rank_smem_raw, &tmA, &tmB);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const SweepRange t = sweep_range(a.R, a.num_n, a.splits);
    const int m0 = t.m0;
    if (warp < 4) {
        if (warp == 0 && lane == 0) rank_produce(&tmA, &tmB, s, m0, t.n_begin * TC_BN, t.n_end - t.n_begin, a.kblocks);
        return;
    }
    const int g = (warp >> 2) - 1;
    int row[2], tgt[2], cnt[2] = {0, 0};
    float st[2];
    const int* ex[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        row[i] = m0 + rank_frag_row(g, i);
        tgt[i] = row[i] < a.R ? a.tid[row[i]] : 0;
        st[i] = tgt[i] ? a.tscore[row[i]] : INFINITY;
        ex[i] = EXCL && row[i] < a.R ? a.excl + (size_t)row[i] * a.E : nullptr;
    }
    const int cb = 2 * (lane & 3);
    int stage = 0;
    uint32_t phase = 0;
    float acc[64];
    mbar_wait(s.a_bar, 0);
    for (int nt = t.n_begin; nt < t.n_end; ++nt) {
        tc_mainloop<0, 0, RANK_STAGES, true>(acc, s.sA, s.sB, s.full_bar, s.empty_bar, 0, a.kblocks, g, stage, phase);
        const int n0 = nt * TC_BN;
        if (n0 > 0 && n0 + TC_BN <= a.C) rank_count_tile<false, EXCL>(acc, st, tgt, ex, a.E, n0, cb, a.C, cnt);
        else rank_count_tile<true, EXCL>(acc, st, tgt, ex, a.E, n0, cb, a.C, cnt);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        int c = cnt[i];
        c += __shfl_xor_sync(0xffffffffu, c, 1);
        c += __shfl_xor_sync(0xffffffffu, c, 2);
        if ((lane & 3) == 0 && tgt[i] && c) atomicAdd(a.cnt + row[i], c);
    }
}

// ------------------------------------------------------------------------------------------------ ranks and metrics
__global__ void __launch_bounds__(256) head_rank_finish_kernel(HeadRankArgs a) {
    pdl_wait();
    const int r = blockIdx.x * 256 + threadIdx.x;
    if (r >= a.R) return;
    const int rank = a.tid[r] ? 1 + a.cnt[r] : 0;
    if (a.ranks) a.ranks[r] = rank;
    if (rank && a.metrics) rank_metrics_add(a.metrics, rank);
}

}  // namespace grb
