// genrec_b200 - Sinkhorn-Knopp balanced assignment of the RQ-VAE's SINKHORN estimator and the k-means centroid update of its codebook
// initialisation (reference: genrec/models/rqvae.py:85-110, :218-241; genrec/modules/kmeans.py:52-99).
//
// Sinkhorn, one launch of ONE thread-block cluster (SK_CLUSTER CTAs, rows split across them):
//   mid = (max d + min d) / 2, amp = (max d - mid) + 1e-5, dn = (d - mid) / amp         fp32, true divisions, global min / max
//   K_ij = exp(-(double)dn_ij / eps)                                                     fp64 from here on
//   v = 1 ; iters x { u = r / (K v + 1e-8) ; v = c / (K^T u + 1e-8) }                    r = (float)(1/B), c = (float)(1/K)
//   ids_i = argmax_j (u_i K_ij) v_j                                                      first index on ties
// One pass over a CTA's rows per iteration: a warp owns whole rows (lane l holds columns l, l + 32, ...), dots the row with v into u_i,
// and accumulates K_ij u_i into its column partials in the same pass.  The warps' partials are added in warp order, the CTAs' partials
// (double-buffered by iteration parity) in CTA-rank order through distributed shared memory, so every CTA derives the same v after one
// cluster barrier per iteration and every sum has a fixed order: ids, u and v are bit-identical from run to run.  A CTA's rows of K sit
// in its shared memory when they fit, otherwise in the caller's workspace (L2-resident at training sizes).
#pragma once
#include <cooperative_groups.h>

#include "common.cuh"

namespace grb {

namespace cg = cooperative_groups;

constexpr int SK_CLUSTER = 16;                 // non-portable cluster size (the host checks that one such cluster fits)
constexpr int SK_THREADS = 512;
constexpr int SK_WARPS = SK_THREADS / 32;
constexpr int SK_KMAX = 256;
constexpr int SK_CPL = SK_KMAX / 32;           // columns per lane
constexpr size_t SK_SMEM_MAX = 227 * 1024;
// v, two parity buffers of column partials, the warps' column partials, min / max
constexpr size_t SK_SMEM_FIXED = (size_t)(SK_KMAX + 2 * SK_KMAX + SK_WARPS * SK_KMAX) * sizeof(double) + 4 * sizeof(float);

struct SinkhornArgs {
    const float* dist;   // [B, K]
    long long B;
    int K, iters, rows;  // rows: rows per CTA
    double eps;
    long long* ids;      // [B]
    double* u_out;       // nullable [B]
    double* v_out;       // nullable [K]
    double* u;           // workspace [B]
    double* kmat;        // workspace [B, K] when the rows of K do not fit shared memory
};

inline size_t sk_rows_per_cta(long long B) { return (size_t)((B + SK_CLUSTER - 1) / SK_CLUSTER); }
inline bool sk_kmat_in_smem(long long B, int K) { return SK_SMEM_FIXED + sk_rows_per_cta(B) * K * sizeof(double) <= SK_SMEM_MAX; }

template <bool KSMEM>
__global__ void __launch_bounds__(SK_THREADS, 1) rq_sinkhorn_kernel(SinkhornArgs a) {
    pdl_wait();
    cg::cluster_group cluster = cg::this_cluster();
    extern __shared__ __align__(16) double sk_smem[];
    double* vs = sk_smem;                                   // [KMAX]
    double* part = vs + SK_KMAX;                            // [2][KMAX]  this CTA's column partials, by iteration parity
    double* wpart = part + 2 * SK_KMAX;                     // [WARPS][KMAX]
    float* mm = reinterpret_cast<float*>(wpart + SK_WARPS * SK_KMAX);   // [2] this CTA's min, max
    double* ks = reinterpret_cast<double*>(mm + 4);         // [rows][K] (KSMEM); mm + 4 keeps 16-byte alignment
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int K = a.K;
    const unsigned rank = cluster.block_rank();
    const long long r0 = (long long)rank * a.rows;
    const int nrows = (int)(a.B - r0 <= 0 ? 0 : (a.B - r0 < a.rows ? a.B - r0 : a.rows));
    const float* d = a.dist + r0 * K;
    double* kb = KSMEM ? ks : a.kmat + r0 * K;
    double* u = a.u + r0;

    // ---- global min / max of dist (exact in any order), exchanged through distributed shared memory
    {
        float lo = INFINITY, hi = -INFINITY;
        for (long long e = tid; e < (long long)nrows * K; e += SK_THREADS) {
            const float x = d[e];
            lo = fminf(lo, x);
            hi = fmaxf(hi, x);
        }
        float* red = reinterpret_cast<float*>(wpart);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o));
            hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o));
        }
        if (lane == 0) { red[warp] = lo; red[SK_WARPS + warp] = hi; }
        __syncthreads();
        if (tid == 0) {
            for (int w = 0; w < SK_WARPS; ++w) { lo = fminf(lo, red[w]); hi = fmaxf(hi, red[SK_WARPS + w]); }
            mm[0] = lo;
            mm[1] = hi;
        }
        cluster.sync();
        lo = INFINITY; hi = -INFINITY;
        for (int r = 0; r < SK_CLUSTER; ++r) {
            const float* rm = cluster.map_shared_rank(mm, r);
            lo = fminf(lo, rm[0]);
            hi = fmaxf(hi, rm[1]);
        }
        // the reference's fp32 arithmetic, round-to-nearest whatever the build's fast-math flags
        const float mid = __fdiv_rn(__fadd_rn(hi, lo), 2.0f);
        const float amp = __fadd_rn(__fsub_rn(hi, mid), 1e-5f);
        for (long long e = tid; e < (long long)nrows * K; e += SK_THREADS) {
            const float dn = __fdiv_rn(__fsub_rn(d[e], mid), amp);
            kb[e] = exp(-(double)dn / a.eps);
        }
        for (int i = tid; i < nrows; i += SK_THREADS) u[i] = 1.0;   // u of zero iterations
        for (int j = tid; j < SK_KMAX; j += SK_THREADS) vs[j] = j < K ? 1.0 : 0.0;
        __syncthreads();
    }
    const double rmarg = (double)(float)(1.0 / (double)a.B);
    const double cmarg = (double)(float)(1.0 / (double)K);

    for (int it = 0; it < a.iters; ++it) {
        double acc[SK_CPL];
#pragma unroll
        for (int c = 0; c < SK_CPL; ++c) acc[c] = 0.0;
        // two rows per step keep twice the loads of K in flight
        for (int lr = warp; lr < nrows; lr += 2 * SK_WARPS) {
            const int lr2 = lr + SK_WARPS;
            const bool two = lr2 < nrows;
            double k0[SK_CPL], k1[SK_CPL];
#pragma unroll
            for (int c = 0; c < SK_CPL; ++c) {
                const int j = lane + 32 * c;
                k0[c] = j < K ? kb[(size_t)lr * K + j] : 0.0;
                k1[c] = (two && j < K) ? kb[(size_t)lr2 * K + j] : 0.0;
            }
            double s0 = 0.0, s1 = 0.0;
#pragma unroll
            for (int c = 0; c < SK_CPL; ++c) {
                const double vj = vs[lane + 32 * c];
                s0 = fma(k0[c], vj, s0);
                s1 = fma(k1[c], vj, s1);
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {     // a butterfly: every lane ends with the same bits
                s0 += __shfl_xor_sync(0xffffffffu, s0, o);
                s1 += __shfl_xor_sync(0xffffffffu, s1, o);
            }
            const double u0 = rmarg / (s0 + 1e-8);
            const double u1 = two ? rmarg / (s1 + 1e-8) : 0.0;
            if (lane == 0 && it == a.iters - 1) {
                u[lr] = u0;
                if (two) u[lr2] = u1;
            }
#pragma unroll
            for (int c = 0; c < SK_CPL; ++c) {
                acc[c] = fma(k0[c], u0, acc[c]);
                acc[c] = fma(k1[c], u1, acc[c]);
            }
        }
#pragma unroll
        for (int c = 0; c < SK_CPL; ++c) wpart[warp * SK_KMAX + lane + 32 * c] = acc[c];
        __syncthreads();
        double* pb = part + (it & 1) * SK_KMAX;
        if (tid < K) {
            double s = 0.0;
            for (int w = 0; w < SK_WARPS; ++w) s += wpart[w * SK_KMAX + tid];
            pb[tid] = s;
        }
        // the partials of iteration it are published; the buffer of parity it & 1 is rewritten only at it + 2, after every CTA has
        // passed the barrier of it + 1, i.e. after every CTA has finished reading it
        cluster.sync();
        if (tid < K) {
            double s = 0.0;
#pragma unroll
            for (int r = 0; r < SK_CLUSTER; ++r) s += cluster.map_shared_rank(pb, r)[tid];
            vs[tid] = cmarg / (s + 1e-8);
        }
        __syncthreads();
    }

    // ---- assignment: argmax_j (u_i K_ij) v_j, first index on ties
    for (int lr = warp; lr < nrows; lr += SK_WARPS) {
        const double ui = u[lr];
        double best = -1.0;    // every P_ij >= 0
        int bj = 0;
#pragma unroll
        for (int c = 0; c < SK_CPL; ++c) {
            const int j = lane + 32 * c;
            if (j < K) {
                const double p = (ui * kb[(size_t)lr * K + j]) * vs[j];
                if (p > best) { best = p; bj = j; }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
            if (ob > best || (ob == best && oj < bj)) { best = ob; bj = oj; }
        }
        if (lane == 0) {
            a.ids[r0 + lr] = bj;
            if (a.u_out) a.u_out[r0 + lr] = ui;
        }
    }
    if (a.v_out && rank == 0)
        for (int j = tid; j < K; j += SK_THREADS) a.v_out[j] = vs[j];
    cluster.sync();   // no CTA leaves while another may still read its shared memory
}

// ------------------------------------------------------------------------------------------------ k-means centroid update
// One CTA per cluster c.  Thread (s, d) walks rows s, s + S, ... (S = KM_THREADS / D) in ascending order and adds column d of every row
// assigned to c in fp64; the S partial sums are then added in order of s.  A non-empty cluster's centroid becomes (float)(sum / count)
// (written in place); an empty one is left unchanged for the host to reseed.  counts[c] and shift[c] = |new - old| go to the caller.
constexpr int KM_THREADS = 256;

__global__ void __launch_bounds__(KM_THREADS) kmeans_update_kernel(const float* x, const long long* assign, long long B, int D,
                                                                   float* cent, int* counts, float* shift) {
    pdl_wait();
    __shared__ double sums[KM_THREADS];
    __shared__ int cnts[KM_THREADS];
    const int c = blockIdx.x, tid = threadIdx.x;
    const int S = KM_THREADS / D, s = tid / D, dcol = tid % D;
    double acc = 0.0;
    int n = 0;
    if (s < S) {
        for (long long i = s; i < B; i += S) {
            if (assign[i] == c) {
                acc += (double)x[i * D + dcol];
                ++n;
            }
        }
    }
    sums[tid] = acc;
    cnts[tid] = n;
    __syncthreads();
    double sq = 0.0;
    int total = 0;
    if (tid < D) {
        double t = 0.0;
        for (int q = 0; q < S; ++q) {
            t += sums[q * D + tid];
            total += cnts[q * D + tid];
        }
        if (total > 0) {
            const float old = cent[(size_t)c * D + tid];
            const float nw = (float)(t / (double)total);
            cent[(size_t)c * D + tid] = nw;
            const double df = (double)nw - (double)old;
            sq = df * df;
        }
    }
    __syncthreads();
    if (tid < D) sums[tid] = sq;
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        for (int j = 0; j < D; ++j) t += sums[j];
        counts[c] = total;
        shift[c] = (float)sqrt(t);
    }
}

}  // namespace grb
