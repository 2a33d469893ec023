// genrec_b200 - what the table-sweeping heads share: the top-k head (head_topk.cuh), the rank head (head_rank.cuh) and the
// candidates head (head_candidates.cuh) sweep the item table without forming the [R, C] logits, one CTA per (128-row tile,
// contiguous range of 128-item tiles), all score with tc_mainloop, and all drop per-row exclusion lists.
//
// Shared-memory rings: rank and candidates keep LN(x) resident and stream table tiles only (RankSmem, rank_cta_init,
// rank_produce below), while top-k's lists and accumulator tile (128 KB) would leave a resident-A ring two table stages, which
// measured slower on an H100 than its three A + B stages at D = 256 and for one-tile ranges.
//
// Exclusion lists: sweep_sort_exclude_kernel turns a row's int64 ids into a sorted int32 list ([R, E], ids outside 1..C-1 ->
// INT_MAX), which sweep_excluded searches.
//
// Total order of every selection: the higher score first, then the lower id (topk_better; topk_key is its order-preserving key
// of the score).
#pragma once
#include <climits>

#include "tc_gemm.cuh"

namespace grb {

constexpr int SWEEP_MAX_EXCLUDE = 16384;
constexpr int SWEEP_SORT_THREADS = 1024;

// total order of every list: the higher score first, then the lower id
GRB_DEVINL bool topk_better(float s, int id, float s2, int id2) { return s > s2 || (s == s2 && id < id2); }

// order-preserving unsigned key of a float score (-0 and +0 compare equal, so they share a key)
GRB_DEVINL unsigned topk_key(float s) {
    unsigned b = __float_as_uint(s);
    if ((b << 1) == 0u) b = 0u;
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// ------------------------------------------------------------------------------------------------ exclusion lists
__global__ void __launch_bounds__(SWEEP_SORT_THREADS) sweep_sort_exclude_kernel(const long long* ex, int E, int P, int C, int* out) {
    pdl_wait();
    extern __shared__ int sort_buf[];           // [P], P = the power of two >= E
    const long long* src = ex + (size_t)blockIdx.x * E;
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const long long v = i < E ? src[i] : 0;
        sort_buf[i] = (v >= 1 && v < C) ? (int)v : INT_MAX;
    }
    __syncthreads();
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = threadIdx.x; t < P / 2; t += blockDim.x) {
                const int i = 2 * t - (t & (stride - 1));          // lower index of the pair, j = i + stride
                const int j = i + stride;
                const bool up = (i & size) == 0;
                const int a = sort_buf[i], b = sort_buf[j];
                if ((a > b) == up) { sort_buf[i] = b; sort_buf[j] = a; }
            }
            __syncthreads();
        }
    }
    int* dst = out + (size_t)blockIdx.x * E;
    for (int i = threadIdx.x; i < E; i += blockDim.x) dst[i] = sort_buf[i];
}

GRB_DEVINL bool sweep_excluded(const int* ex, int E, int id) {
    int lo = 0, hi = E;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(ex + mid) < id) lo = mid + 1;
        else hi = mid;
    }
    return lo < E && __ldg(ex + lo) == id;
}

// ------------------------------------------------------------------------------------------------ work of a CTA
// This CTA's work: row tile m0 and item tiles n_begin .. n_end-1 of range `split`.  blockIdx.x = split * num_m + row tile, so the
// CTAs that read the same item range for different row tiles run side by side and a table tile comes from HBM once.
struct SweepRange {
    int m0, split, n_begin, n_end;
};
GRB_DEVINL SweepRange sweep_range(int R, int num_n, int splits) {
    const int num_m = (R + TC_BM - 1) / TC_BM;
    SweepRange t;
    t.m0 = (blockIdx.x % num_m) * TC_BM;
    t.split = blockIdx.x / num_m;
    t.n_begin = (int)((long long)t.split * num_n / splits);
    t.n_end = (int)((long long)(t.split + 1) * num_n / splits);
    return t;
}

// ------------------------------------------------------------------------------------------------ resident-A ring
// A CTA keeps one row tile: its LN(x) operand (up to D / 64 = 4 k-blocks of 16 KB) is loaded once and stays in shared memory, and
// the ring carries table tiles only, 8 stages of 16 KB.
constexpr int RANK_STAGES = 8;
constexpr int RANK_MAX_KBLOCKS = 4;
constexpr int RANK_SMEM_BYTES = (RANK_MAX_KBLOCKS + RANK_STAGES) * TC_TILE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
struct RankSmem {
    unsigned char *sA, *sB;                      // sA: [kblocks] resident A tiles ; sB: [RANK_STAGES] ring of B tiles
    uint64_t *full_bar, *empty_bar, *a_bar;
};
// carve the shared memory, initialise the barriers and wait for the previous kernel
GRB_DEVINL RankSmem rank_cta_init(unsigned char* raw, const CUtensorMap* tmA, const CUtensorMap* tmB) {
    unsigned char* base = raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
    RankSmem s;
    s.sA = base;
    s.sB = base + RANK_MAX_KBLOCKS * TC_TILE_BYTES;
    s.full_bar = reinterpret_cast<uint64_t*>(base + (RANK_MAX_KBLOCKS + RANK_STAGES) * TC_TILE_BYTES);
    s.empty_bar = s.full_bar + RANK_STAGES;
    s.a_bar = s.empty_bar + RANK_STAGES;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(tmA);
        tma_prefetch_desc(tmB);
        for (int i = 0; i < RANK_STAGES; ++i) {
            mbar_init(&s.full_bar[i], 1);
            mbar_init(&s.empty_bar[i], 2);
        }
        mbar_init(s.a_bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    return s;
}
// TMA producer (one lane): row tile m0 of A once, then the B tiles starting at rows b0, b0 + 128, ... (ntiles of them)
GRB_DEVINL void rank_produce(const CUtensorMap* tmA, const CUtensorMap* tmB, const RankSmem& s, int m0, int b0, int ntiles, int kblocks) {
    mbar_expect_tx(s.a_bar, kblocks * TC_TILE_BYTES);
    for (int kb = 0; kb < kblocks; ++kb) tma_load_2d(s.sA + kb * TC_TILE_BYTES, tmA, kb * TC_BK, m0, s.a_bar);
    int stage = 0;
    uint32_t phase = 0;
    for (int n = 0; n < ntiles; ++n) {
        for (int kb = 0; kb < kblocks; ++kb) {
            mbar_wait(&s.empty_bar[stage], phase ^ 1);
            mbar_expect_tx(&s.full_bar[stage], TC_TILE_BYTES);
            tma_load_2d(s.sB + stage * TC_TILE_BYTES, tmB, kb * TC_BK, b0 + n * TC_BN, &s.full_bar[stage]);
            if (++stage == RANK_STAGES) { stage = 0; phase ^= 1; }
        }
    }
}
// tile row of accumulator row i (0, 1) of this consumer thread: wgmma D fragment rows lane / 4 and lane / 4 + 8 of the warp's 16
GRB_DEVINL int rank_frag_row(int g, int i) { return g * 64 + ((threadIdx.x >> 5) & 3) * 16 + ((threadIdx.x & 31) >> 2) + 8 * i; }

}  // namespace grb
