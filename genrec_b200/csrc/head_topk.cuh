// genrec_b200 - top-k items of the tied-embedding head without the [R, C] logits (grb_head_topk).
//
//   scores[r, :], items[r, :] = the k best items of LN(x[r]) . E^T, best first, in the total order (score desc, item id asc);
//   item 0 (padding) and the ids of the row's exclusion list never appear; missing slots hold (-inf, 0).
//
// Launches after the LayerNorm and the exclusion sort (head_sweep.cuh):
//   head_topk_kernel           TMA + mbarrier + wgmma (tc_mainloop of tc_gemm.cuh, K = D), one CTA per (row tile, item range) as
//                              sweep_range (head_sweep.cuh) assigns them: the CTA walks its contiguous range of 128-item tiles,
//                              and for each row of its tile keeps a sorted list of k (score, id) in the shared memory
//                              tc_gemm_kernel uses for output staging.  The list's k-th score is the row's threshold, so a score
//                              that cannot enter costs one compare; the few that pass are merged into the list by one warp at
//                              once.  Ids are visited in increasing order, so "pass when strictly greater than the k-th score"
//                              is the tie rule exactly.
//   topk_merge_kernel          one warp per row: k-way merge of the per-range lists under the same total order
// Every score is the fp32 accumulator of the same wgmma sequence grb_head_logits runs for that (row, item), so the scores are
// bit-identical to its logits, and the total order makes the result independent of how the items are split across CTAs.
#pragma once
#include "head_sweep.cuh"

namespace grb {

constexpr int TOPK_MAX_K = 64;
constexpr int TOPK_MAX_SPLITS = 256;            // item ranges per row tile (the merge keeps one cursor per range in shared memory)
constexpr int TOPK_MERGE_ROWS = 4;              // rows (warps) per merge CTA
static_assert(TOPK_MAX_K * TC_BM * 8 <= TC_STAGE_OUT_BYTES, "the per-row lists live in the output staging buffer");

struct HeadTopkArgs {
    int R, C, k, E;
    int splits, num_n, kblocks;
    const int* excl;            // [R, E] sorted int32 (INT_MAX = ignored entry), or null
    float* cand_s;              // [R, splits, k]
    int* cand_i;                // [R, splits, k]
};

// One warp merges the candidates ok[q] (score v[q], item id[q]; lane holds 4) into the row's sorted list ls / li [k] in shared
// memory.  When more than k candidates pass, those with at least k others of strictly higher score cannot enter and are dropped
// first (the k-th largest key, found bit by bit with ballots).  Then every entry's new slot is its rank in the union, i.e. the
// number of entries of the union better than it, counted while each candidate in turn is broadcast to the warp.  The total order
// makes the ranks distinct, so the stores below never collide; whatever ranks k or beyond drops out.
GRB_DEVINL void topk_merge_row(float* ls, int* li, int k, const float (&v)[4], const int (&id)[4], bool (&ok)[4], int lane) {
    int q_all = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) q_all += __popc(__ballot_sync(0xffffffffu, ok[q]));
    if (q_all > k) {
        unsigned key[4], t = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) key[q] = ok[q] ? topk_key(v[q]) : 0u;
        for (int bit = 31; bit >= 0; --bit) {
            const unsigned t2 = t | (1u << bit);
            int cnt = 0;
#pragma unroll
            for (int q = 0; q < 4; ++q) cnt += __popc(__ballot_sync(0xffffffffu, key[q] >= t2));
            if (cnt >= k) t = t2;
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) ok[q] = ok[q] && key[q] >= t;
    }
    const float s0 = lane < k ? ls[lane] : -INFINITY, s1 = lane + 32 < k ? ls[lane + 32] : -INFINITY;
    const int i0 = lane < k ? li[lane] : INT_MAX, i1 = lane + 32 < k ? li[lane + 32] : INT_MAX;
    int rank0 = lane, rank1 = lane + 32;
    int rk[4] = {0, 0, 0, 0};
#pragma unroll
    for (int q2 = 0; q2 < 4; ++q2) {
        unsigned m = __ballot_sync(0xffffffffu, ok[q2]);
        while (m) {
            const int b = __ffs(m) - 1;
            m &= m - 1;
            const float cs = __shfl_sync(0xffffffffu, v[q2], b);
            const int ci = __shfl_sync(0xffffffffu, id[q2], b);
            rank0 += topk_better(cs, ci, s0, i0);
            rank1 += topk_better(cs, ci, s1, i1);
            const int in_list = __popc(__ballot_sync(0xffffffffu, lane < k && topk_better(s0, i0, cs, ci))) +
                                __popc(__ballot_sync(0xffffffffu, lane + 32 < k && topk_better(s1, i1, cs, ci)));
            if (lane == b) rk[q2] += in_list;
#pragma unroll
            for (int q = 0; q < 4; ++q) rk[q] += topk_better(cs, ci, v[q], id[q]);
        }
    }
    __syncwarp();                                // every lane has read the old list
    if (lane < k && rank0 < k) { ls[rank0] = s0; li[rank0] = i0; }
    if (lane + 32 < k && rank1 < k) { ls[rank1] = s1; li[rank1] = i1; }
#pragma unroll
    for (int q = 0; q < 4; ++q)
        if (ok[q] && rk[q] < k) { ls[rk[q]] = v[q]; li[rk[q]] = id[q]; }
    __syncwarp();
}

// ------------------------------------------------------------------------------------------------ scoring + per-range lists
// Warp roles as tc_gemm_kernel; in the selection step warp w of consumer warpgroup g owns rows 64 g + 16 w .. +15 of the tile
// (among the rows its warpgroup's wgmma produced) and their lists.
__global__ void __launch_bounds__(TC_THREADS, 1)
    head_topk_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, HeadTopkArgs a) {
    extern __shared__ unsigned char topk_smem_raw[];
    unsigned char* base = topk_smem_raw + ((1024u - (smem_u32(topk_smem_raw) & 1023u)) & 1023u);
    unsigned char* sA = base;
    unsigned char* sB = base + TC_STAGES * TC_TILE_BYTES;
    float* lsc = reinterpret_cast<float*>(base + 2 * TC_STAGES * TC_TILE_BYTES);   // [128][TOPK_MAX_K] list scores, one row per tile row
    int* lid = reinterpret_cast<int*>(lsc + TOPK_MAX_K * TC_BM);                    // [128][TOPK_MAX_K] list ids
    float* sAcc = reinterpret_cast<float*>(base + 2 * TC_STAGES * TC_TILE_BYTES + TC_STAGE_OUT_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(base + 2 * TC_STAGES * TC_TILE_BYTES + TC_STAGE_OUT_BYTES + TC_ACC_BYTES);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + TC_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const SweepRange t = sweep_range(a.R, a.num_n, a.splits);
    const int m0 = t.m0;

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < TC_STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 2);
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();

    if (warp < 4) {
        // ===================================================================== TMA producer
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int nt = t.n_begin; nt < t.n_end; ++nt) {
                for (int kb = 0; kb < a.kblocks; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_expect_tx(&full_bar[stage], 2 * TC_TILE_BYTES);
                    tma_load_2d(sA + stage * TC_TILE_BYTES, &tmA, kb * TC_BK, m0, &full_bar[stage]);
                    tma_load_2d(sB + stage * TC_TILE_BYTES, &tmB, kb * TC_BK, nt * TC_BN, &full_bar[stage]);
                    if (++stage == TC_STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
        return;
    }
    // ===================================================================== consumers: MMA + selection
    const int g = (warp >> 2) - 1;
    const int r0 = g * 64 + (warp & 3) * 16;     // this warp's 16 tile rows (inside the 64 its warpgroup's wgmma produced)
    const int k = a.k;
    for (int j = lane; j < 16 * TOPK_MAX_K; j += 32) {
        lsc[r0 * TOPK_MAX_K + j] = -INFINITY;
        lid[r0 * TOPK_MAX_K + j] = 0;
    }
    __syncwarp();
    int stage = 0;
    uint32_t phase = 0;
    float acc[64];
    for (int nt = t.n_begin; nt < t.n_end; ++nt) {
        tc_mainloop<0, 0, TC_STAGES>(acc, sA, sB, full_bar, empty_bar, 0, a.kblocks, g, stage, phase);
        wg_bar_sync(g);                          // this warpgroup's selection of the previous tile has read sAcc
        tc_acc_store(sAcc, acc, g);
        wg_bar_sync(g);
        const int n0 = nt * TC_BN;
#pragma unroll 1
        for (int i = 0; i < 16; ++i) {
            const int r = r0 + i, row = m0 + r;
            if (row >= a.R) break;
            const float thr = lsc[r * TOPK_MAX_K + k - 1];   // the list's k-th score
            float v[4];
            int id[4];
            bool ok[4];
            unsigned any = 0;
#pragma unroll
            for (int q = 0; q < 4; ++q) {        // lane holds columns lane + 32 q
                const int c = 32 * q + lane;
                v[q] = sAcc[r * TC_BN + (((c >> 2) ^ (r & 7)) << 2) + (c & 3)];
                id[q] = n0 + c;
                ok[q] = v[q] > thr && id[q] != 0 && id[q] < a.C;
                any |= __ballot_sync(0xffffffffu, ok[q]);
            }
            if (!any) continue;
            if (a.excl) {
                const int* ex = a.excl + (size_t)row * a.E;
                any = 0;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    if (ok[q] && sweep_excluded(ex, a.E, id[q])) ok[q] = false;
                    any |= __ballot_sync(0xffffffffu, ok[q]);
                }
                if (!any) continue;
            }
            topk_merge_row(lsc + r * TOPK_MAX_K, lid + r * TOPK_MAX_K, k, v, id, ok, lane);
        }
    }
    for (int j = lane; j < 16 * k; j += 32) {
        const int i = j / k, s = j - i * k, row = m0 + r0 + i;
        if (row < a.R) {
            a.cand_s[((size_t)row * a.splits + t.split) * k + s] = lsc[(r0 + i) * TOPK_MAX_K + s];
            a.cand_i[((size_t)row * a.splits + t.split) * k + s] = lid[(r0 + i) * TOPK_MAX_K + s];
        }
    }
}

// ------------------------------------------------------------------------------------------------ merge of the ranges
__global__ void __launch_bounds__(32 * TOPK_MERGE_ROWS) topk_merge_kernel(const float* cand_s, const int* cand_i, int R, int splits, int k,
                                                                          float* scores, long long* items) {
    pdl_wait();
    __shared__ int cursor[TOPK_MERGE_ROWS][TOPK_MAX_SPLITS];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row = blockIdx.x * TOPK_MERGE_ROWS + w;
    if (row >= R) return;
    int* cur = cursor[w];
    for (int i = lane; i < splits; i += 32) cur[i] = 0;
    __syncwarp();
    const float* cs = cand_s + (size_t)row * splits * k;
    const int* ci = cand_i + (size_t)row * splits * k;
    // this lane's best list head over ranges lane, lane + 32, ...
    float bs = -INFINITY;
    int bid = INT_MAX, bl = -1;
    auto rescan = [&]() {
        bs = -INFINITY; bid = INT_MAX; bl = -1;
        for (int i = lane; i < splits; i += 32) {
            const int p = cur[i];
            if (p < k) {
                const float s = cs[i * k + p];
                const int id = ci[i * k + p];
                if (topk_better(s, id, bs, bid)) { bs = s; bid = id; bl = i; }
            }
        }
    };
    rescan();
    for (int o = 0; o < k; ++o) {
        float ws = bs;
        int wid = bid, wl = lane;
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            const float s2 = __shfl_xor_sync(0xffffffffu, ws, off);
            const int id2 = __shfl_xor_sync(0xffffffffu, wid, off);
            const int l2 = __shfl_xor_sync(0xffffffffu, wl, off);
            if (topk_better(s2, id2, ws, wid) || (s2 == ws && id2 == wid && l2 < wl)) { ws = s2; wid = id2; wl = l2; }
        }
        if (lane == 0) {
            scores[(size_t)row * k + o] = ws;
            items[(size_t)row * k + o] = ws == -INFINITY ? 0 : wid;
        }
        if (lane == wl) {
            ++cur[bl];
            rescan();
        }
        __syncwarp();
    }
}

}  // namespace grb
