// genrec_b200 - RQ-VAE residual nearest-codebook search (reference: genrec/models/rqvae.py:185-199, :397-412).
//
//   for level l:  id_l = argmin_k ( |r|^2 + |c_k|^2 - 2 r.c_k )  (first index on ties) ;  r <- r - c_{id_l}
//
// No tensor cores by specification: FP32 FMA on the CUDA cores.  One thread owns one item row (its residual lives in
// registers for all levels); the level's codebook sits in shared memory and every lane reads the SAME code word at the
// same time (a broadcast, conflict-free), so the inner loop is 4 FFMA per 16-byte LDS.  Two code words are processed
// per iteration for ILP.  HBM traffic per item: D*4 B in, levels*8 B out (+ optional embeddings / residuals / loss).
#pragma once
#include "common.cuh"

namespace grb {

constexpr int RQ_THREADS = 256;

struct RqArgs {
    const float* x;          // [N, D] latent
    const float* codebooks;  // [levels, K, D]
    long long* ids;          // [N, levels]
    float* emb;              // nullable [N, D, levels]   (reference layout, rqvae.py:408)
    float* res;              // nullable [N, D, levels]   residual BEFORE each level (rqvae.py:400, :409)
    float* loss;             // nullable [N]  sum_l (1 + w) * |r_l - e_l|^2   (loss.py:75-77)
    float* res_out;          // nullable [N, D] final residual
    long long N;
    int K, levels;
    float commitment;
};

// ROWS item rows per thread (register tile): one broadcast LDS.128 of a code word feeds 4 * ROWS FFMA, which moves the
// inner loop from shared-memory-issue bound (ROWS = 1: 1 LDS per 4 FFMA) to FMA bound (ROWS = 2).
template <int D, int ROWS>
__global__ void __launch_bounds__(RQ_THREADS) rq_residual_argmin_kernel(RqArgs a) {
    pdl_wait();
    extern __shared__ __align__(16) float rq_smem[];
    float* cb = rq_smem;             // [K][D]
    float* cn = rq_smem + a.K * D;   // [K] squared norms
    const int tid = threadIdx.x;
    long long row[ROWS];
    bool live[ROWS];
    float r[ROWS][D];
#pragma unroll
    for (int q = 0; q < ROWS; ++q) {
        row[q] = ((long long)blockIdx.x * ROWS + q) * RQ_THREADS + tid;
        live[q] = row[q] < a.N;
        if (live[q]) {
#pragma unroll
            for (int j = 0; j < D; j += 4) {
                float4 v = *reinterpret_cast<const float4*>(a.x + row[q] * D + j);
                r[q][j] = v.x; r[q][j + 1] = v.y; r[q][j + 2] = v.z; r[q][j + 3] = v.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < D; ++j) r[q][j] = 0.f;
        }
    }
    float loss[ROWS];
#pragma unroll
    for (int q = 0; q < ROWS; ++q) loss[q] = 0.f;

    for (int l = 0; l < a.levels; ++l) {
        __syncthreads();
        const float* g = a.codebooks + (size_t)l * a.K * D;
        for (int i = tid * 4; i < a.K * D; i += RQ_THREADS * 4)
            *reinterpret_cast<float4*>(cb + i) = *reinterpret_cast<const float4*>(g + i);
        __syncthreads();
        for (int k = tid; k < a.K; k += RQ_THREADS) {
            float s = 0.f;
            for (int j = 0; j < D; ++j) s = fmaf(cb[k * D + j], cb[k * D + j], s);
            cn[k] = s;
        }
        __syncthreads();

        float xn[ROWS], best[ROWS];
        int best_k[ROWS];
#pragma unroll
        for (int q = 0; q < ROWS; ++q) {
            xn[q] = 0.f;
#pragma unroll
            for (int j = 0; j < D; ++j) xn[q] = fmaf(r[q][j], r[q][j], xn[q]);
            if (a.res && live[q]) {
#pragma unroll
                for (int j = 0; j < D; ++j) a.res[(row[q] * D + j) * a.levels + l] = r[q][j];
            }
            best[q] = INFINITY;
            best_k[q] = 0;
        }
        for (int k = 0; k < a.K; k += 2) {
            float d0[ROWS], d1[ROWS];
#pragma unroll
            for (int q = 0; q < ROWS; ++q) d0[q] = d1[q] = 0.f;
            const float4* c0 = reinterpret_cast<const float4*>(cb + k * D);
            const float4* c1 = reinterpret_cast<const float4*>(cb + (k + 1) * D);
#pragma unroll
            for (int j = 0; j < D / 4; ++j) {
                const float4 u = c0[j], w = c1[j];
#pragma unroll
                for (int q = 0; q < ROWS; ++q) {
                    d0[q] = fmaf(r[q][4 * j], u.x, d0[q]); d0[q] = fmaf(r[q][4 * j + 1], u.y, d0[q]);
                    d0[q] = fmaf(r[q][4 * j + 2], u.z, d0[q]); d0[q] = fmaf(r[q][4 * j + 3], u.w, d0[q]);
                    d1[q] = fmaf(r[q][4 * j], w.x, d1[q]); d1[q] = fmaf(r[q][4 * j + 1], w.y, d1[q]);
                    d1[q] = fmaf(r[q][4 * j + 2], w.z, d1[q]); d1[q] = fmaf(r[q][4 * j + 3], w.w, d1[q]);
                }
            }
            const float n0 = cn[k], n1 = cn[k + 1];
#pragma unroll
            for (int q = 0; q < ROWS; ++q) {
                const float dist0 = (xn[q] + n0) - 2.f * d0[q];
                const float dist1 = (xn[q] + n1) - 2.f * d1[q];
                if (dist0 < best[q]) { best[q] = dist0; best_k[q] = k; }
                if (dist1 < best[q]) { best[q] = dist1; best_k[q] = k + 1; }
            }
        }
#pragma unroll
        for (int q = 0; q < ROWS; ++q) {
            float sq = 0.f;
            const float* cw = cb + best_k[q] * D;
#pragma unroll
            for (int j = 0; j < D; ++j) {
                const float e = cw[j];
                if (a.emb && live[q]) a.emb[(row[q] * D + j) * a.levels + l] = e;
                r[q][j] -= e;
                sq = fmaf(r[q][j], r[q][j], sq);
            }
            loss[q] += sq + a.commitment * sq;
            if (live[q]) a.ids[row[q] * a.levels + l] = best_k[q];
        }
    }
#pragma unroll
    for (int q = 0; q < ROWS; ++q) {
        if (!live[q]) continue;
        if (a.loss) a.loss[row[q]] = loss[q];
        if (a.res_out) {
#pragma unroll
            for (int j = 0; j < D; j += 4)
                *reinterpret_cast<float4*>(a.res_out + row[q] * D + j) = make_float4(r[q][j], r[q][j + 1], r[q][j + 2], r[q][j + 3]);
        }
    }
}

// ------------------------------------------------------------------------------------------------ split variant
// The same arithmetic (dot products accumulated in the same order, the same (|r|^2 + |c|^2) - 2 r.c expression, strict '<' on
// an ascending code index), but a row is scanned by FOUR threads, each walking a quarter of the codes; the quarters meet
// through two shuffles (lower index wins ties, so the first-index rule of torch.min survives).  N = 12,101 items become 189
// CTAs instead of 48, and a row's serial chain is 64 codes instead of 256.  Lanes are laid out quarter-major (lane = q * 8 +
// row): the 8 lanes of a shared-memory phase read ONE code word (a broadcast), so the LDS.128 stays conflict-free.
// Optional outputs in the reference's [N, D, levels] layout are staged in shared memory per row and written once, as whole
// contiguous rows with 16-byte stores (writing them level by level is a stride-`levels` scatter at ~5 % of HBM speed).
constexpr int RQ_SPLIT = 4;
constexpr int RQ_ROWS_PER_CTA = RQ_THREADS / RQ_SPLIT;   // x ROWS

template <int D, int ROWS, bool STAGE>
__global__ void __launch_bounds__(RQ_THREADS) rq_residual_argmin_split_kernel(RqArgs a) {
    pdl_wait();
    extern __shared__ __align__(16) float rq_smem[];
    float* cb = rq_smem;             // [K][D]
    float* cn = rq_smem + a.K * D;   // [K] squared norms
    float* st_emb = cn + ((a.K + 3) & ~3);                                   // [rows of the CTA][D * levels]   (STAGE)
    float* st_res = st_emb + (size_t)RQ_ROWS_PER_CTA * ROWS * D * a.levels;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int q = lane >> 3;                         // code quarter
    const int rl = warp * 8 + (lane & 7);            // row slot inside the CTA (0 .. 63), x ROWS
    const int kq = a.K / RQ_SPLIT;                   // codes per quarter (K % 8 == 0 checked by the host)
    const long long row0 = (long long)blockIdx.x * RQ_ROWS_PER_CTA * ROWS;
    long long row[ROWS];
    bool live[ROWS];
    float r[ROWS][D];
#pragma unroll
    for (int w = 0; w < ROWS; ++w) {
        row[w] = row0 + (long long)w * RQ_ROWS_PER_CTA + rl;
        live[w] = row[w] < a.N;
        if (live[w]) {
#pragma unroll
            for (int j = 0; j < D; j += 4) {
                float4 v = *reinterpret_cast<const float4*>(a.x + row[w] * D + j);
                r[w][j] = v.x; r[w][j + 1] = v.y; r[w][j + 2] = v.z; r[w][j + 3] = v.w;
            }
        } else {
#pragma unroll
            for (int j = 0; j < D; ++j) r[w][j] = 0.f;
        }
    }
    float loss[ROWS];
#pragma unroll
    for (int w = 0; w < ROWS; ++w) loss[w] = 0.f;
    constexpr int JQ = D / RQ_SPLIT;   // columns of a row each of its four threads writes out

    for (int l = 0; l < a.levels; ++l) {
        __syncthreads();
        const float* g = a.codebooks + (size_t)l * a.K * D;
        for (int i = tid * 4; i < a.K * D; i += RQ_THREADS * 4)
            *reinterpret_cast<float4*>(cb + i) = *reinterpret_cast<const float4*>(g + i);
        __syncthreads();
        for (int k = tid; k < a.K; k += RQ_THREADS) {
            float s = 0.f;
            for (int j = 0; j < D; ++j) s = fmaf(cb[k * D + j], cb[k * D + j], s);
            cn[k] = s;
        }
        __syncthreads();

        float xn[ROWS], best[ROWS];
        int best_k[ROWS];
#pragma unroll
        for (int w = 0; w < ROWS; ++w) {
            xn[w] = 0.f;
#pragma unroll
            for (int j = 0; j < D; ++j) xn[w] = fmaf(r[w][j], r[w][j], xn[w]);
            if (a.res) {
                // each of the row's four threads writes a quarter of the columns; the quarter is selected by an unrolled compare
                // so that r[][] keeps compile-time indices (a run-time index would push the whole array to local memory)
#pragma unroll
                for (int qq = 0; qq < RQ_SPLIT; ++qq) {
                    if (q != qq) continue;
#pragma unroll
                    for (int jj = 0; jj < JQ; ++jj) {
                        const int j = qq * JQ + jj;
                        if (STAGE) st_res[((size_t)(w * RQ_ROWS_PER_CTA + rl) * D + j) * a.levels + l] = r[w][j];
                        else if (live[w]) a.res[(row[w] * D + j) * a.levels + l] = r[w][j];
                    }
                }
            }
            best[w] = INFINITY;
            best_k[w] = 0;
        }
        const int k_lo = q * kq;
        for (int k = k_lo; k < k_lo + kq; k += 2) {
            float d0[ROWS], d1[ROWS];
#pragma unroll
            for (int w = 0; w < ROWS; ++w) d0[w] = d1[w] = 0.f;
            const float4* c0 = reinterpret_cast<const float4*>(cb + k * D);
            const float4* c1 = reinterpret_cast<const float4*>(cb + (k + 1) * D);
#pragma unroll
            for (int j = 0; j < D / 4; ++j) {
                const float4 u = c0[j], v = c1[j];
#pragma unroll
                for (int w = 0; w < ROWS; ++w) {
                    d0[w] = fmaf(r[w][4 * j], u.x, d0[w]); d0[w] = fmaf(r[w][4 * j + 1], u.y, d0[w]);
                    d0[w] = fmaf(r[w][4 * j + 2], u.z, d0[w]); d0[w] = fmaf(r[w][4 * j + 3], u.w, d0[w]);
                    d1[w] = fmaf(r[w][4 * j], v.x, d1[w]); d1[w] = fmaf(r[w][4 * j + 1], v.y, d1[w]);
                    d1[w] = fmaf(r[w][4 * j + 2], v.z, d1[w]); d1[w] = fmaf(r[w][4 * j + 3], v.w, d1[w]);
                }
            }
            const float n0 = cn[k], n1 = cn[k + 1];
#pragma unroll
            for (int w = 0; w < ROWS; ++w) {
                const float dist0 = (xn[w] + n0) - 2.f * d0[w];
                const float dist1 = (xn[w] + n1) - 2.f * d1[w];
                if (dist0 < best[w]) { best[w] = dist0; best_k[w] = k; }
                if (dist1 < best[w]) { best[w] = dist1; best_k[w] = k + 1; }
            }
        }
        // the four quarters of a row sit in lanes (lane & 7) + {0, 8, 16, 24}
#pragma unroll
        for (int w = 0; w < ROWS; ++w) {
#pragma unroll
            for (int o = 8; o <= 16; o <<= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best[w], o);
                const int ok = __shfl_xor_sync(0xffffffffu, best_k[w], o);
                if (ob < best[w] || (ob == best[w] && ok < best_k[w])) { best[w] = ob; best_k[w] = ok; }
            }
        }
#pragma unroll
        for (int w = 0; w < ROWS; ++w) {
            float sq = 0.f;
            const float* cw = cb + best_k[w] * D;
#pragma unroll
            for (int j = 0; j < D; ++j) {
                const float e = cw[j];
                r[w][j] -= e;
                sq = fmaf(r[w][j], r[w][j], sq);
            }
            if (a.emb) {
#pragma unroll
                for (int jj = 0; jj < JQ; ++jj) {
                    const int j = q * JQ + jj;
                    if (STAGE) st_emb[((size_t)(w * RQ_ROWS_PER_CTA + rl) * D + j) * a.levels + l] = cw[j];
                    else if (live[w]) a.emb[(row[w] * D + j) * a.levels + l] = cw[j];
                }
            }
            loss[w] += sq + a.commitment * sq;
            if (live[w] && q == 0) a.ids[row[w] * a.levels + l] = best_k[w];
        }
    }
#pragma unroll
    for (int w = 0; w < ROWS; ++w) {
        if (!live[w] || q != 0) continue;
        if (a.loss) a.loss[row[w]] = loss[w];
        if (a.res_out) {
#pragma unroll
            for (int j = 0; j < D; j += 4)
                *reinterpret_cast<float4*>(a.res_out + row[w] * D + j) = make_float4(r[w][j], r[w][j + 1], r[w][j + 2], r[w][j + 3]);
        }
    }
    if (STAGE && (a.emb || a.res)) {
        // staged rows -> global: ROWS slabs of RQ_ROWS_PER_CTA consecutive rows, each slab one contiguous span
        __syncthreads();
        const int per_row = D * a.levels;              // floats, a multiple of 4
#pragma unroll
        for (int w = 0; w < ROWS; ++w) {
            const long long first = row0 + (long long)w * RQ_ROWS_PER_CTA;
            long long nrows = a.N - first;
            if (nrows <= 0) continue;
            if (nrows > RQ_ROWS_PER_CTA) nrows = RQ_ROWS_PER_CTA;
            const size_t nfl = (size_t)nrows * per_row;
            const float* s_e = st_emb + (size_t)w * RQ_ROWS_PER_CTA * per_row;
            const float* s_r = st_res + (size_t)w * RQ_ROWS_PER_CTA * per_row;
            for (size_t i = (size_t)tid * 4; i < nfl; i += RQ_THREADS * 4) {
                if (a.emb) *reinterpret_cast<float4*>(a.emb + (size_t)first * per_row + i) = *reinterpret_cast<const float4*>(s_e + i);
                if (a.res) *reinterpret_cast<float4*>(a.res + (size_t)first * per_row + i) = *reinterpret_cast<const float4*>(s_r + i);
            }
        }
    }
}


// ------------------------------------------------------------------------------------------------ register-blocked tile variant
// The two kernels above feed 4 (or 8) FFMA per 16-byte shared-memory load; an LDS.128 delivers 512 B to the register file and the
// SM moves 128 B per clock, so they are bound by the shared-memory -> register path at ~25 % (50 %) of the FMA rate, and at the
// catalogue size (N = 12,101) additionally by one serial chain of 3 x 256 (or 64) codes per thread on a third of the SMs.
// This variant is the distance "GEMM" on the CUDA cores: a CTA owns 128 item rows; the residual tile and the level's codebook sit
// TRANSPOSED in shared memory (rT[d][row], cT[d][code]); thread (rg, cg) accumulates an 8-row x 16-code block of dot products in
// registers - per d: 2 + 4 LDS.128 feed 128 FFMA.  Every (row, code) dot product is still ONE fmaf chain over d = 0 .. D-1
// and the distance is still (|r|^2 + |c|^2) - 2 r.c with strict '<' over ascending code indices, so ids are bit-identical to the
// kernels above (tests/test_rq_gpu.py).  The 16 threads that share a row meet through 4 shuffle steps (lower index wins ties).
// Outputs in the reference's [N, D, levels] layout are staged per tile and written as one contiguous span.
constexpr int RQT_ROWS = 128;             // rows per CTA: every CTA transposes the level's codebook for itself, so fewer, larger tiles
constexpr int RQT_THREADS = 256;          // 16 code groups x 16 row groups
constexpr int RQT_RLD = RQT_ROWS + 4;     // row pitch of the transposed residual tile (floats); +4 keeps the float4 loads 16-byte aligned
template <int D>
__global__ void __launch_bounds__(RQT_THREADS, 1) rq_residual_argmin_tile_kernel(RqArgs a) {
    pdl_wait();
    extern __shared__ __align__(16) float rq_smem[];
    const int KLD = a.K + 4;
    float* rT = rq_smem;                               // [D][RQT_RLD]   residual, transposed
    float* cT = rT + D * RQT_RLD;                      // [D][KLD]       codebook level, transposed
    float* cn = cT + D * KLD;                          // [K]            |c|^2
    float* xn = cn + ((a.K + 3) & ~3);                 // [rows]         |r|^2
    float* lossv = xn + RQT_ROWS;                      // [rows]
    int* sid = reinterpret_cast<int*>(lossv + RQT_ROWS);          // [rows][levels] chosen codes
    float* st_emb = reinterpret_cast<float*>(sid + ((RQT_ROWS * a.levels + 3) & ~3));   // [rows][D * levels] (emb or res requested)
    float* st_res = st_emb + (size_t)RQT_ROWS * D * a.levels;
    const bool stage = a.emb != nullptr || a.res != nullptr;
    const int tid = threadIdx.x;
    const int cg = tid & 15, rg = tid >> 4;            // code group (16 codes), row group (8 rows)
    const long long row0 = (long long)blockIdx.x * RQT_ROWS;
    const int nrows = (int)((a.N - row0) < RQT_ROWS ? (a.N - row0) : RQT_ROWS);

    // ---- residual tile: coalesced float4 reads of [rows][D], transposed into rT (rows past N are zeros)
    for (int e = tid; e < RQT_ROWS * (D / 4); e += RQT_THREADS) {
        const int r = e / (D / 4), d4 = e % (D / 4);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (r < nrows) v = *reinterpret_cast<const float4*>(a.x + (row0 + r) * D + 4 * d4);
        rT[(4 * d4) * RQT_RLD + r] = v.x; rT[(4 * d4 + 1) * RQT_RLD + r] = v.y;
        rT[(4 * d4 + 2) * RQT_RLD + r] = v.z; rT[(4 * d4 + 3) * RQT_RLD + r] = v.w;
    }
    __syncthreads();
    if (tid < RQT_ROWS) {
        float s = 0.f;
#pragma unroll 8
        for (int j = 0; j < D; ++j) s = fmaf(rT[j * RQT_RLD + tid], rT[j * RQT_RLD + tid], s);
        xn[tid] = s;
        lossv[tid] = 0.f;
    }

    for (int l = 0; l < a.levels; ++l) {
        __syncthreads();
        const float* g = a.codebooks + (size_t)l * a.K * D;
        for (int e = tid; e < a.K * (D / 4); e += RQT_THREADS) {
            const int k = e / (D / 4), d4 = e % (D / 4);
            const float4 v = *reinterpret_cast<const float4*>(g + (size_t)k * D + 4 * d4);
            cT[(4 * d4) * KLD + k] = v.x; cT[(4 * d4 + 1) * KLD + k] = v.y;
            cT[(4 * d4 + 2) * KLD + k] = v.z; cT[(4 * d4 + 3) * KLD + k] = v.w;
        }
        __syncthreads();
        for (int k = tid; k < a.K; k += RQT_THREADS) {
            float s = 0.f;
#pragma unroll 8
            for (int j = 0; j < D; ++j) s = fmaf(cT[j * KLD + k], cT[j * KLD + k], s);
            cn[k] = s;
        }
        __syncthreads();

        float best[8];
        int best_k[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) { best[i] = INFINITY; best_k[i] = 0; }
        // rows of this thread: rg*8 + {0..7}; codes per 256-code pass: q*64 + cg*4 + {0..3}, q = 0..3
        for (int kb = 0; kb < a.K; kb += 256) {
            float acc[8][16];
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 16; ++j) acc[i][j] = 0.f;
#pragma unroll 2
            for (int d = 0; d < D; ++d) {
                const float* rrow = rT + d * RQT_RLD + rg * 8;
                const float* crow = cT + d * KLD + kb;
                const float4 a0 = *reinterpret_cast<const float4*>(rrow);
                const float4 a1 = *reinterpret_cast<const float4*>(rrow + 4);
                const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float4 b = *reinterpret_cast<const float4*>(crow + q * 64 + cg * 4);   // codes k .. k+3
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        acc[i][4 * q] = fmaf(av[i], b.x, acc[i][4 * q]);
                        acc[i][4 * q + 1] = fmaf(av[i], b.y, acc[i][4 * q + 1]);
                        acc[i][4 * q + 2] = fmaf(av[i], b.z, acc[i][4 * q + 2]);
                        acc[i][4 * q + 3] = fmaf(av[i], b.w, acc[i][4 * q + 3]);
                    }
                }
            }
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float x2 = xn[rg * 8 + i];
#pragma unroll
                for (int j = 0; j < 16; ++j) {            // ascending code index inside the thread: q-major, then the 4 of a chunk
                    const int k = kb + (j >> 2) * 64 + cg * 4 + (j & 3);
                    const float dist = (x2 + cn[k]) - 2.f * acc[i][j];
                    if (dist < best[i]) { best[i] = dist; best_k[i] = k; }
                }
            }
        }
        // the 16 code groups of a row group are the 16 lanes of a half warp: lexicographic (distance, index) minimum
#pragma unroll
        for (int i = 0; i < 8; ++i) {
#pragma unroll
            for (int o = 1; o < 16; o <<= 1) {
                const float ob = __shfl_xor_sync(0xffffffffu, best[i], o);
                const int ok = __shfl_xor_sync(0xffffffffu, best_k[i], o);
                if (ob < best[i] || (ob == best[i] && ok < best_k[i])) { best[i] = ob; best_k[i] = ok; }
            }
            if (cg == 0) sid[(rg * 8 + i) * a.levels + l] = best_k[i];
        }
        __syncthreads();
        if (stage) {
            // residual BEFORE the level and the chosen code word -> staging, all threads, lanes along d (stride `levels` in the
            // [row][d][level] layout: conflict-free for levels coprime with 32, e.g. 3)
            for (int e = tid; e < RQT_ROWS * D; e += RQT_THREADS) {
                const int r = e / D, j = e % D;
                st_res[(size_t)e * a.levels + l] = rT[j * RQT_RLD + r];
                st_emb[(size_t)e * a.levels + l] = cT[j * KLD + sid[r * a.levels + l]];
            }
            __syncthreads();
        }
        // residual update, one thread per row (the same serial fmaf chain as the other kernels: |r_new|^2 is next level's |r|^2)
        if (tid < RQT_ROWS) {
            const int k = sid[tid * a.levels + l];
            float sq = 0.f;
#pragma unroll 8
            for (int j = 0; j < D; ++j) {
                float r = rT[j * RQT_RLD + tid] - cT[j * KLD + k];
                sq = fmaf(r, r, sq);
                rT[j * RQT_RLD + tid] = r;
            }
            xn[tid] = sq;
            lossv[tid] += sq + a.commitment * sq;
        }
    }
    __syncthreads();
    // ---- outputs
    for (int e = tid; e < nrows * a.levels; e += RQT_THREADS) a.ids[row0 * a.levels + e] = sid[e];
    if (a.loss && tid < nrows) a.loss[row0 + tid] = lossv[tid];
    if (a.res_out) {
        for (int e = tid; e < nrows * D; e += RQT_THREADS) a.res_out[row0 * D + e] = rT[(e % D) * RQT_RLD + e / D];
    }
    if (stage) {
        const size_t nfl = (size_t)nrows * D * a.levels;    // one contiguous span of the [N, D, levels] tensors, a multiple of 4 floats
        for (size_t i = (size_t)tid * 4; i < nfl; i += RQT_THREADS * 4) {
            if (a.emb) *reinterpret_cast<float4*>(a.emb + (size_t)row0 * D * a.levels + i) = *reinterpret_cast<const float4*>(st_emb + i);
            if (a.res) *reinterpret_cast<float4*>(a.res + (size_t)row0 * D * a.levels + i) = *reinterpret_cast<const float4*>(st_res + i);
        }
    }
}
inline size_t rq_tile_smem_bytes(int D, int K, int levels, bool stage) {
    size_t fl = (size_t)D * RQT_RLD + (size_t)D * (K + 4) + ((K + 3) & ~3) + 2 * RQT_ROWS + ((RQT_ROWS * levels + 3) & ~3);
    if (stage) fl += (size_t)2 * RQT_ROWS * D * levels;
    return fl * sizeof(float);
}

}  // namespace grb
