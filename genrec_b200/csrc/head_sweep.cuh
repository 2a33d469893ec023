// genrec_b200 - what the top-k head (head_topk.cuh) and the rank head (head_rank.cuh) share: both sweep the item table without
// forming the [R, C] logits, one CTA per (128-row tile, contiguous range of 128-item tiles), both score with tc_mainloop, and both
// drop per-row exclusion lists.  Their shared-memory rings differ: rank keeps LN(x) resident and streams table tiles only, while
// top-k's lists and accumulator tile (128 KB) would leave a resident-A ring two table stages, which measured slower on an H100
// than its three A + B stages at D = 256 and for one-tile ranges.
//
// Exclusion lists: sweep_sort_exclude_kernel turns a row's int64 ids into a sorted int32 list ([R, E], ids outside 1..C-1 ->
// INT_MAX), which sweep_excluded searches.
#pragma once
#include <climits>

#include "tc_gemm.cuh"

namespace grb {

constexpr int SWEEP_MAX_EXCLUDE = 16384;
constexpr int SWEEP_SORT_THREADS = 1024;

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

}  // namespace grb
