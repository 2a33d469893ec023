// genrec_b200 - up to 2048 best items of the tied-embedding head without the [R, C] logits (grb_head_candidates for k > 64;
// k <= 64 runs the top-k head of head_topk.cuh).
//
//   scores[r, :], items[r, :] = the k best items of LN(x[r]) . E^T, best first, in the total order (score desc, item id asc);
//   item 0 (padding) and the ids of the row's exclusion list never appear; missing slots hold (-inf, 0).
//
// A pair (s, id) has the 64-bit key (topk_key(s) << 32) | ~id, so "better in the total order" is "larger key" and every key is
// distinct.  Launches after the LayerNorm and the exclusion sort (head_sweep.cuh), the same sequence whatever the data:
//   head_cand_sweep_kernel<BOUND>     one CTA per (row tile, item range) on the resident-A ring (RankSmem): each consumer thread
//                                     keeps the CAND_M best eligible pairs of each of its two accumulator rows in registers and
//                                     writes their keys to lists [R, splits, 4, CAND_M].  These are distinct eligible items.
//   head_cand_threshold_kernel        one CTA per row: tau = the k-th largest listed key (radix select), or 0 when fewer than k
//                                     are listed.  At least k eligible items have a key >= tau, so the k best all do.
//   head_cand_sweep_kernel<COLLECT>   re-scores the table and appends every eligible pair with key >= tau to the row's buffer
//                                     [R, cap] (one atomicAdd per row and quad of lanes); the row's count goes on past cap.
//   8 x (head_cand_sweep_kernel<HIST>, head_cand_digit_kernel)
//                                     a row whose count passed cap lost pairs, so its exact k-th key is found byte by byte, most
//                                     significant first: the sweep histograms the next byte of the keys >= tau that share the
//                                     bytes found so far, and the digit kernel picks the byte holding the k-th.  CTAs and rows
//                                     without an overflowed row return at once.
//   head_cand_sweep_kernel<RECOLLECT> collects the overflowed rows again with tau = their exact k-th key: exactly k pairs.
//   head_cand_select_kernel           one CTA per row: bitonic sort of the row's pairs by key in shared memory, the first k out.
// Every score is the fp32 accumulator of the wgmma sequence grb_head_logits runs for that (row, item) (tc_mainloop), so the scores
// are bit-identical to its logits; the answer is the unique top k of the total order, whatever the split of the items.
#pragma once
#include "head_sweep.cuh"

namespace grb {

constexpr int CAND_MAX_K = 2048;
constexpr int CAND_M = 8;                      // pairs per accumulator row and consumer thread in the bound sweep
constexpr int CAND_LIST_PER_K = 2;             // the bound sweep lists at least 2 k pairs per row (where the catalog allows)
constexpr int CAND_CAP_PER_K = 4;              // a row's collect buffer holds 4 k pairs
constexpr int CAND_RADIX_PASSES = 8;           // bytes of a key
constexpr int CAND_SELECT_THREADS = 1024;
constexpr int CAND_DIGIT_THREADS = 256;

enum CandPass { CAND_BOUND, CAND_COLLECT, CAND_HIST, CAND_RECOLLECT };

struct HeadCandArgs {
    int R, C, k, E, cap;
    int splits, num_n, kblocks;
    const int* excl;                           // [R, E] sorted int32 (INT_MAX = ignored entry), or null
    unsigned long long* lists;                 // [R, splits, 4, CAND_M] keys of the bound sweep (0 = empty slot)
    unsigned long long* tau;                   // [R] collect threshold key (0: every eligible item)
    unsigned long long* prefix;                // [R] bytes of the exact k-th key found so far (overflowed rows)
    int* krem;                                 // [R] rank of the k-th key among the keys >= tau that share prefix
    int* cnt;                                  // [R] pairs at or above tau (counts on past cap)
    int* redo;                                 // [R] 1: the row overflowed and is collected again
    int* hist;                                 // [R, 256]
    float* buf_s;                              // [R, cap]
    int* buf_i;                                // [R, cap]
};

GRB_DEVINL unsigned long long cand_key(float s, int id) { return ((unsigned long long)topk_key(s) << 32) | (unsigned)~id; }
// the score of a key's upper half (+0 for the key -0 and +0 share)
GRB_DEVINL float cand_key_score(unsigned hi) { return __uint_as_float((hi & 0x80000000u) ? (hi & 0x7fffffffu) : ~hi); }

// One warp: the byte d whose bin of h[256] (counts per byte value) holds the k-th largest key, and in k that key's rank inside the
// bin.  Lane l reads bins 255 - 8 l .. 248 - 8 l; a scan over the lanes finds the lane, and that lane finds the bin.
GRB_DEVINL int cand_pick_byte(const int* h, int& k, int lane) {
    int c[8], sum = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) { c[q] = h[255 - 8 * lane - q]; sum += c[q]; }
    int incl = sum;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, incl, off);
        if (lane >= off) incl += o;
    }
    const unsigned hit = __ballot_sync(0xffffffffu, incl >= k);
    const int L = hit ? __ffs(hit) - 1 : 31;
    int kk = k - __shfl_sync(0xffffffffu, incl - sum, L), q = 7;
    bool found = false;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        if (!found) {
            if (c[j] >= kk || j == 7) { found = true; q = j; }
            else kk -= c[j];
        }
    }
    k = __shfl_sync(0xffffffffu, kk, L);
    return 255 - 8 * L - __shfl_sync(0xffffffffu, q, L);
}

template <bool EXCL>
GRB_DEVINL bool cand_eligible(const int* ex, int E, int id, int C) {
    return id >= 1 && id < C && !(EXCL && sweep_excluded(ex, E, id));
}

// ------------------------------------------------------------------------------------------------ the sweeps, per table tile
// Column 8 j + e of this thread's accumulators is item n0 + 8 j + e (n0 includes the thread's column base); accumulator row i
// holds acc[4 j + 2 i + e].  Along the sweep a thread meets its items in increasing id order.

// BOUND: insert into the row's best-first register list.  An equal score already listed has the lower id, so a pair enters only
// above a strictly lower score and goes below every equal one.
template <bool EXCL>
GRB_DEVINL void cand_bound_tile(const float (&acc)[64], const bool (&on)[2], const int* const (&ex)[2], int E, int n0, int C,
                                float (&ls)[2][CAND_M], int (&li)[2][CAND_M]) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        if (!on[i]) continue;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const float v = acc[4 * j + 2 * i + e];
                const int id = n0 + 8 * j + e;
                if (v > ls[i][CAND_M - 1] && cand_eligible<EXCL>(ex[i], E, id, C)) {
#pragma unroll
                    for (int q = CAND_M - 1; q > 0; --q) {
                        const bool down = v > ls[i][q - 1];
                        li[i][q] = down ? li[i][q - 1] : (v > ls[i][q] ? id : li[i][q]);
                        ls[i][q] = down ? ls[i][q - 1] : (v > ls[i][q] ? v : ls[i][q]);
                    }
                    if (v > ls[i][0]) { ls[i][0] = v; li[i][0] = id; }
                }
            }
        }
    }
}

// COLLECT / RECOLLECT: append the pairs at or above (ts, ti) to the row's buffer.  The 4 lanes of a row (a quad) reserve their
// places with one atomicAdd; places past cap are counted but not written.
template <bool EXCL>
GRB_DEVINL void cand_collect_tile(const float (&acc)[64], const bool (&on)[2], const int* const (&ex)[2], int E, int n0, int C,
                                  const float (&ts)[2], const int (&ti)[2], const int (&row)[2], const HeadCandArgs& a) {
    unsigned mask[2] = {0u, 0u};
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        if (!on[i]) continue;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const float v = acc[4 * j + 2 * i + e];
                const int id = n0 + 8 * j + e;
                if ((v > ts[i] || (v == ts[i] && id <= ti[i])) && cand_eligible<EXCL>(ex[i], E, id, C)) mask[i] |= 1u << (2 * j + e);
            }
        }
    }
    if (!__any_sync(0xffffffffu, (mask[0] | mask[1]) != 0u)) return;
    const int ql = threadIdx.x & 3;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int n = __popc(mask[i]);
        int incl = n, o = __shfl_up_sync(0xffffffffu, incl, 1, 4);
        if (ql >= 1) incl += o;
        o = __shfl_up_sync(0xffffffffu, incl, 2, 4);
        if (ql >= 2) incl += o;
        int base = 0;
        if (ql == 3 && incl) base = atomicAdd(a.cnt + row[i], incl);
        int pos = __shfl_sync(0xffffffffu, base, 3, 4) + incl - n;
        if (!n) continue;
        float* bs = a.buf_s + (size_t)row[i] * a.cap;
        int* bi = a.buf_i + (size_t)row[i] * a.cap;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                if ((mask[i] >> (2 * j + e)) & 1u) {
                    if (pos < a.cap) { bs[pos] = acc[4 * j + 2 * i + e]; bi[pos] = n0 + 8 * j + e; }
                    ++pos;
                }
            }
        }
    }
}

// HIST: add byte `shift / 8` of every eligible key >= tau whose higher bytes equal prefix to the row's histogram.  Runs of one
// byte value (a flat table gives long ones) are added with one atomicAdd each.
template <bool EXCL>
GRB_DEVINL void cand_hist_tile(const float (&acc)[64], const bool (&on)[2], const int* const (&ex)[2], int E, int n0, int C,
                               const unsigned long long (&tau)[2], const unsigned long long (&pre)[2], int shift, const int (&row)[2],
                               int* hist) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        if (!on[i]) continue;
        int* h = hist + (size_t)row[i] * 256;
        int cur = 0, run = 0;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int id = n0 + 8 * j + e;
                const unsigned long long key = cand_key(acc[4 * j + 2 * i + e], id);
                if (key >= tau[i] && (shift == 56 || (key >> (shift + 8)) == pre[i]) && cand_eligible<EXCL>(ex[i], E, id, C)) {
                    const int d = (int)(key >> shift) & 255;
                    if (run && d != cur) { atomicAdd(h + cur, run); run = 0; }
                    cur = d;
                    ++run;
                }
            }
        }
        if (run) atomicAdd(h + cur, run);
    }
}

// One CTA per (row tile, item range) as sweep_range assigns them, on the resident-A ring; `pass` is the radix pass of HIST.
template <int PASS, bool EXCL>
__global__ void __launch_bounds__(TC_THREADS, 1)
    head_cand_sweep_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, HeadCandArgs a, int pass) {
    extern __shared__ unsigned char cand_smem_raw[];
    const SweepRange t = sweep_range(a.R, a.num_n, a.splits);
    const int m0 = t.m0;
    auto refining = [&](int r) { return PASS == CAND_HIST ? a.cnt[r] > a.cap : a.redo[r] != 0; };
    if (PASS == CAND_HIST || PASS == CAND_RECOLLECT) {
        // only rows that overflowed: a CTA without one leaves before its first load (the producer too)
        pdl_wait();
        const int r = m0 + (int)threadIdx.x;
        if (!__syncthreads_or(threadIdx.x < TC_BM && r < a.R && refining(r))) return;
    }
    const RankSmem s = rank_cta_init(cand_smem_raw, &tmA, &tmB);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp < 4) {
        if (warp == 0 && lane == 0) rank_produce(&tmA, &tmB, s, m0, t.n_begin * TC_BN, t.n_end - t.n_begin, a.kblocks);
        return;
    }
    const int g = (warp >> 2) - 1;
    int row[2];
    bool on[2];
    const int* ex[2];
    float ts[2];
    int ti[2];
    unsigned long long tau[2], pre[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        row[i] = m0 + rank_frag_row(g, i);
        on[i] = row[i] < a.R && (PASS == CAND_BOUND || PASS == CAND_COLLECT || refining(row[i]));
        ex[i] = EXCL && on[i] ? a.excl + (size_t)row[i] * a.E : nullptr;
        tau[i] = PASS != CAND_BOUND && on[i] ? a.tau[row[i]] : 0ull;
        pre[i] = PASS == CAND_HIST && on[i] ? a.prefix[row[i]] : 0ull;
        // tau as a pair: key 0 lets every eligible item pass
        ts[i] = tau[i] ? cand_key_score((unsigned)(tau[i] >> 32)) : -INFINITY;
        ti[i] = tau[i] ? (int)~(unsigned)tau[i] : INT_MAX;
    }
    float ls[2][CAND_M];
    int li[2][CAND_M];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int q = 0; q < CAND_M; ++q) { ls[i][q] = -INFINITY; li[i][q] = 0; }
    const int cb = 2 * (lane & 3), shift = 56 - 8 * pass;
    int stage = 0;
    uint32_t phase = 0;
    float acc[64];
    mbar_wait(s.a_bar, 0);
    for (int nt = t.n_begin; nt < t.n_end; ++nt) {
        tc_mainloop<0, 0, RANK_STAGES, true>(acc, s.sA, s.sB, s.full_bar, s.empty_bar, 0, a.kblocks, g, stage, phase);
        const int n0 = nt * TC_BN + cb;
        if (PASS == CAND_BOUND) cand_bound_tile<EXCL>(acc, on, ex, a.E, n0, a.C, ls, li);
        else if (PASS == CAND_HIST) cand_hist_tile<EXCL>(acc, on, ex, a.E, n0, a.C, tau, pre, shift, row, a.hist);
        else cand_collect_tile<EXCL>(acc, on, ex, a.E, n0, a.C, ts, ti, row, a);
    }
    if (PASS == CAND_BOUND) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            if (!on[i]) continue;
            unsigned long long* dst = a.lists + (((size_t)row[i] * a.splits + t.split) * 4 + (lane & 3)) * CAND_M;
#pragma unroll
            for (int q = 0; q < CAND_M; ++q) dst[q] = ls[i][q] == -INFINITY ? 0ull : cand_key(ls[i][q], li[i][q]);
        }
    }
}

// ------------------------------------------------------------------------------------------------ threshold of a row
// The k-th largest of the row's listed keys, one byte per pass through a shared histogram; it also resets the row's state.
__global__ void __launch_bounds__(256) head_cand_threshold_kernel(HeadCandArgs a) {
    pdl_wait();
    __shared__ int h[256];
    __shared__ int s_k, s_n;
    __shared__ unsigned long long s_pre;
    const int r = blockIdx.x, n = a.splits * 4 * CAND_M;
    const unsigned long long* L = a.lists + (size_t)r * n;
    h[threadIdx.x] = 0;
    a.hist[(size_t)r * 256 + threadIdx.x] = 0;
    if (threadIdx.x == 0) {
        s_n = 0;
        a.cnt[r] = 0;
        a.redo[r] = 0;
        a.prefix[r] = 0ull;
        a.krem[r] = a.k;
    }
    __syncthreads();
    int c = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) c += L[i] != 0ull;
    if (c) atomicAdd(&s_n, c);
    __syncthreads();
    if (s_n < a.k) {
        if (threadIdx.x == 0) a.tau[r] = 0ull;
        return;
    }
    unsigned long long pre = 0ull;
    int k = a.k;
    for (int p = 0; p < CAND_RADIX_PASSES; ++p) {
        const int shift = 56 - 8 * p;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const unsigned long long key = L[i];
            if (key != 0ull && (p == 0 || (key >> (shift + 8)) == pre)) atomicAdd(&h[(key >> shift) & 255], 1);
        }
        __syncthreads();
        if (threadIdx.x < 32) {
            const int d = cand_pick_byte(h, k, threadIdx.x);
            if (threadIdx.x == 0) {
                s_pre = (pre << 8) | (unsigned)d;
                s_k = k;
            }
        }
        __syncthreads();
        pre = s_pre;
        k = s_k;
        h[threadIdx.x] = 0;
        __syncthreads();
    }
    if (threadIdx.x == 0) a.tau[r] = pre;
}

// ------------------------------------------------------------------------------------------------ radix digit of an overflowed row
// One warp per row, after the histogram of pass `pass`: the byte holding the row's k-th key joins prefix.  After the last pass
// prefix is that key, which becomes the row's tau for the recollect sweep.
__global__ void __launch_bounds__(CAND_DIGIT_THREADS) head_cand_digit_kernel(HeadCandArgs a, int pass) {
    pdl_wait();
    const int r = blockIdx.x * (CAND_DIGIT_THREADS / 32) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= a.R || a.cnt[r] <= a.cap) return;
    int* h = a.hist + (size_t)r * 256;
    int k = a.krem[r];
    const int d = cand_pick_byte(h, k, lane);
    __syncwarp();
    for (int i = lane; i < 256; i += 32) h[i] = 0;
    if (lane) return;
    const unsigned long long pre = (a.prefix[r] << 8) | (unsigned)d;
    if (pass + 1 < CAND_RADIX_PASSES) {
        a.prefix[r] = pre;
        a.krem[r] = k;
    } else {
        a.tau[r] = pre;
        a.cnt[r] = 0;
        a.redo[r] = 1;
    }
}

// ------------------------------------------------------------------------------------------------ final order
// One CTA per row: the row's n pairs (n <= cap) sorted by key, best first, by a bitonic sort over the power of two >= n in shared
// memory ([P] keys, then [P] scores, P = the power of two >= cap); slots k > n get (-inf, 0).
__global__ void __launch_bounds__(CAND_SELECT_THREADS) head_cand_select_kernel(HeadCandArgs a, float* scores, long long* items) {
    pdl_wait();
    extern __shared__ unsigned long long cand_sort_buf[];
    const int r = blockIdx.x;
    const int n = min(a.cnt[r], a.cap);
    int P = 1;
    while (P < n) P <<= 1;
    unsigned long long* key = cand_sort_buf;
    float* sc = reinterpret_cast<float*>(cand_sort_buf + P);
    const float* bs = a.buf_s + (size_t)r * a.cap;
    const int* bi = a.buf_i + (size_t)r * a.cap;
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const float s = i < n ? bs[i] : -INFINITY;
        key[i] = i < n ? cand_key(s, bi[i]) : 0ull;
        sc[i] = s;
    }
    __syncthreads();
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = threadIdx.x; t < P / 2; t += blockDim.x) {
                const int i = 2 * t - (t & (stride - 1));          // lower index of the pair, j = i + stride
                const int j = i + stride;
                const bool down = (i & size) == 0;
                const unsigned long long ki = key[i], kj = key[j];
                if ((ki < kj) == down && ki != kj) {
                    key[i] = kj; key[j] = ki;
                    const float f = sc[i]; sc[i] = sc[j]; sc[j] = f;
                }
            }
            __syncthreads();
        }
    }
    for (int o = threadIdx.x; o < a.k; o += blockDim.x) {
        const float s = o < n ? sc[o] : -INFINITY;
        scores[(size_t)r * a.k + o] = s;
        items[(size_t)r * a.k + o] = s == -INFINITY ? 0 : (int)~(unsigned)key[o];
    }
}

}  // namespace grb
