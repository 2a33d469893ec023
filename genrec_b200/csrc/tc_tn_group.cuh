// genrec_b200 - grouped weight-gradient GEMM:  for each problem p:  Out_p[M_p, N_p] += A_p^T B_p   (A_p stored [K, M_p],
// B_p stored [K, N_p], both row-major bf16; K = number of tokens).  One persistent launch covers all the weight
// gradients of an HSTU layer (dWp, dW1, dW2): every problem is split along K into enough work items to fill the chip,
// a CTA walks its items back to back (the TMA producer runs ahead into the next item while the consumers reduce the
// last one).  The k-split partial tiles go to device scratch; tn_finish_kernel sums them in split order and adds the sums to the
// flat fp32 gradient buffer with 16-byte vector reductions (red.global.add.v4.f32), so the result does not depend on timing.
#pragma once
#include "tc_gemm.cuh"

namespace grb {

constexpr int TN_MAX_PROBLEMS = 4;

struct TnProblem {
    int M, N, K;
    int num_m, num_n, splits, kb_total, kb_per_split;
    int work_begin;  // first global work-item index of this problem
    int part_begin;  // first partial tile of this problem in the scratch (splits > 1)
    float* out;
    int ldo;
};
struct TnGroupParams {
    CUtensorMap tmA[TN_MAX_PROBLEMS];
    CUtensorMap tmB[TN_MAX_PROBLEMS];
    TnProblem p[TN_MAX_PROBLEMS];
    int nprob;
    int total_work;
    float* part;     // split-K partial tiles [128][128] fp32 (problems with splits > 1)
};


struct TnItem {
    int prob, m0, n0, kb0, kb1;
};
GRB_DEVINL TnItem tn_decode(const TnGroupParams& P, int w) {
    int pi = 0;
#pragma unroll
    for (int i = 1; i < TN_MAX_PROBLEMS; ++i)
        if (i < P.nprob && w >= P.p[i].work_begin) pi = i;
    const TnProblem& q = P.p[pi];
    const int local = w - q.work_begin;
    const int split = local % q.splits, tile = local / q.splits;
    TnItem it;
    it.prob = pi;
    it.m0 = (tile / q.num_n) * TC_BM;
    it.n0 = (tile % q.num_n) * TC_BN;
    it.kb0 = split * q.kb_per_split;
    it.kb1 = min(q.kb_total, it.kb0 + q.kb_per_split);
    return it;
}

constexpr int TN_STAGES = 4;

__global__ void __launch_bounds__(TC_THREADS, 1) tc_tn_group_kernel(const __grid_constant__ TnGroupParams P) {
    extern __shared__ unsigned char tn_smem_raw[];
    unsigned char* base = tn_smem_raw + ((1024u - (smem_u32(tn_smem_raw) & 1023u)) & 1023u)   /* offset from the __shared__ array: keeps the shared address space (LDS / STS) */;
    unsigned char* sA = base;
    unsigned char* sB = base + TN_STAGES * TC_TILE_BYTES;
    float* sAcc = reinterpret_cast<float*>(base + 2 * TN_STAGES * TC_TILE_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(base + 2 * TN_STAGES * TC_TILE_BYTES + TC_ACC_BYTES);
    uint64_t* full_bar = bars;
    uint64_t* empty_bar = bars + TN_STAGES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (warp == 0 && lane == 0) {
        for (int i = 0; i < P.nprob; ++i) { tma_prefetch_desc(&P.tmA[i]); tma_prefetch_desc(&P.tmB[i]); }
        for (int s = 0; s < TN_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 2); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();  // prologue above overlaps the previous kernel's tail

    if (warp < 4) {
        if (warp == 0 && lane == 0) {
            int stage = 0; uint32_t phase = 0;
            for (int w = blockIdx.x; w < P.total_work; w += gridDim.x) {
                const TnItem it = tn_decode(P, w);
                const CUtensorMap* ta = &P.tmA[it.prob];
                const CUtensorMap* tb = &P.tmB[it.prob];
                for (int kb = it.kb0; kb < it.kb1; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_expect_tx(&full_bar[stage], 2 * TC_TILE_BYTES);
                    unsigned char* a_dst = sA + stage * TC_TILE_BYTES;
                    unsigned char* b_dst = sB + stage * TC_TILE_BYTES;
                    const int k0 = kb * TC_BK;
                    tma_load_2d(a_dst, ta, it.m0, k0, &full_bar[stage]);
                    tma_load_2d(a_dst + TC_TILE_BYTES / 2, ta, it.m0 + 64, k0, &full_bar[stage]);
                    tma_load_2d(b_dst, tb, it.n0, k0, &full_bar[stage]);
                    tma_load_2d(b_dst + TC_TILE_BYTES / 2, tb, it.n0 + 64, k0, &full_bar[stage]);
                    if (++stage == TN_STAGES) { stage = 0; phase ^= 1; }
                }
            }
        }
    } else {
        const int g = (warp >> 2) - 1, wi = warp & 3;
        const int sub = g * 2 + (wi & 1), cq = wi >> 1;
        int stage = 0; uint32_t phase = 0;
        float acc[64];
        for (int w = blockIdx.x; w < P.total_work; w += gridDim.x) {
            const TnItem it = tn_decode(P, w);
            tc_mainloop<1, 1, TN_STAGES>(acc, sA, sB, full_bar, empty_bar, it.kb0, it.kb1, g, stage, phase);
            wg_bar_sync(g);
            tc_acc_store(sAcc, acc, g);
            wg_bar_sync(g);
            const TnProblem& q = P.p[it.prob];
            const int r = sub * 32 + lane;
            if (q.splits > 1) {
                // the partial tile of this k-split; tn_finish_kernel sums the splits of every tile in split order
                float* part = P.part + (size_t)(q.part_begin + (w - q.work_begin)) * (TC_BM * TC_BN);
#pragma unroll 1
                for (int c = cq * TC_EPI_CPW; c < (cq + 1) * TC_EPI_CPW; ++c) {
                    float v[32];
                    tc_acc_load32(sAcc, r, c, v);
#pragma unroll
                    for (int j = 0; j < 8; ++j)
                        *reinterpret_cast<float4*>(part + r * TC_BN + c * 32 + 4 * j) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                }
                continue;
            }
            // one k-split: the only add to these elements in this launch
            const int row = it.m0 + r;
#pragma unroll 1
            for (int c = cq * TC_EPI_CPW; c < (cq + 1) * TC_EPI_CPW; ++c) {
                float v[32];
                tc_acc_load32(sAcc, r, c, v);
                const int col0 = it.n0 + c * 32;
                if (row < q.M && col0 < q.N) {
                    float* dst = q.out + (size_t)row * q.ldo + col0;
                    if (col0 + 32 <= q.N && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
#pragma unroll
                        for (int j = 0; j < 8; ++j) red_add_v4(dst + 4 * j, v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                    } else {
                        for (int i = 0; i < 32; ++i)
                            if (col0 + i < q.N) atomicAdd(dst + i, v[i]);
                    }
                }
            }
        }
    }
}

// Out_p[tile] += sum of the tile's k-split partials in split order (TN_FINISH_SLABS CTAs per output tile, 16-byte vector reductions)
constexpr int TN_FINISH_SLABS = 16;   // 8 rows x 128 columns = one float4 per thread
__global__ void __launch_bounds__(256) tn_finish_kernel(const __grid_constant__ TnGroupParams P) {
    pdl_wait();
    // the tiles of the problems with splits > 1, problem after problem
    int t = blockIdx.x / TN_FINISH_SLABS, pi = 0;
    for (; pi < P.nprob; ++pi) {
        if (P.p[pi].splits == 1) continue;
        const int tiles = P.p[pi].num_m * P.p[pi].num_n;
        if (t < tiles) break;
        t -= tiles;
    }
    if (pi >= P.nprob) return;
    const TnProblem& q = P.p[pi];
    const int m0 = (t / q.num_n) * TC_BM, n0 = (t % q.num_n) * TC_BN;
    const float* part = P.part + (size_t)(q.part_begin + t * q.splits) * (TC_BM * TC_BN);
    const int f = (blockIdx.x % TN_FINISH_SLABS) * 256 + threadIdx.x;
    const int r = f / (TC_BN / 4), c = 4 * (f % (TC_BN / 4));
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
    for (int sp = 0; sp < q.splits; ++sp) {
        const float4 v = reinterpret_cast<const float4*>(part + (size_t)sp * (TC_BM * TC_BN))[f];
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    const int row = m0 + r, col = n0 + c;
    if (row >= q.M || col >= q.N) return;
    float* dst = q.out + (size_t)row * q.ldo + col;
    if (col + 4 <= q.N && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
        red_add_v4(dst, s.x, s.y, s.z, s.w);
    } else {
        const float sv[4] = {s.x, s.y, s.z, s.w};
        for (int e = 0; e < 4 && col + e < q.N; ++e) atomicAdd(dst + e, sv[e]);
    }
}

constexpr int TN_SMEM_BYTES = 2 * TN_STAGES * TC_TILE_BYTES + TC_ACC_BYTES + 1024 + 256;

struct TnSpec {
    const bf16* A; const bf16* B; float* out;
    int M, N, K, lda, ldb, ldo;
};

// work split of a launch: every problem gets a share of (2 work items per SM) proportional to its FLOPs; returns the floats of
// split-K partial tiles the launch needs (the `part` scratch of launch_tc_tn_group)
inline size_t tn_plan(TnGroupParams& P, const TnSpec* specs, int n, int num_sms) {
    memset(&P, 0, sizeof(P));
    P.nprob = n;
    double total = 0;
    for (int i = 0; i < n; ++i) total += (double)specs[i].M * specs[i].N * specs[i].K;
    int work = 0, parts = 0;
    for (int i = 0; i < n; ++i) {
        const TnSpec& s = specs[i];
        TnProblem& q = P.p[i];
        q.M = s.M; q.N = s.N; q.K = s.K; q.out = s.out; q.ldo = s.ldo;
        q.num_m = (s.M + TC_BM - 1) / TC_BM;
        q.num_n = (s.N + TC_BN - 1) / TC_BN;
        q.kb_total = (s.K + TC_BK - 1) / TC_BK;
        const int tiles = q.num_m * q.num_n;
        int want_items = (int)(2.0 * num_sms * ((double)s.M * s.N * s.K / total) + 0.5);
        int splits = (want_items + tiles - 1) / tiles;
        if (splits < 1) splits = 1;
        int max_splits = q.kb_total / 4 > 0 ? q.kb_total / 4 : 1;  // at least 4 k-blocks per item
        if (splits > max_splits) splits = max_splits;
        q.kb_per_split = (q.kb_total + splits - 1) / splits;
        q.splits = (q.kb_total + q.kb_per_split - 1) / q.kb_per_split;
        q.work_begin = work;
        q.part_begin = q.splits > 1 ? parts : -1;
        work += tiles * q.splits;
        if (q.splits > 1) parts += tiles * q.splits;
    }
    P.total_work = work;
    return (size_t)parts * (TC_BM * TC_BN);
}
inline size_t tn_part_floats(const TnSpec* specs, int n, int num_sms) {
    TnGroupParams P;
    return n < 1 || n > TN_MAX_PROBLEMS ? 0 : tn_plan(P, specs, n, num_sms);
}

// part: tn_part_floats(specs, n, num_sms) floats of scratch
inline cudaError_t launch_tc_tn_group(const TnSpec* specs, int n, int num_sms, float* part, cudaStream_t st) {
    if (n < 1 || n > TN_MAX_PROBLEMS) return cudaErrorInvalidValue;
    TnGroupParams P;
    const size_t need = tn_plan(P, specs, n, num_sms);
    if (need > 0 && part == nullptr) return cudaErrorInvalidValue;
    P.part = part;
    for (int i = 0; i < n; ++i) {
        const TnSpec& s = specs[i];
        if (!make_tmap_bf16(&P.tmA[i], s.A, s.K, s.M, s.lda, 64, TC_BK) || !make_tmap_bf16(&P.tmB[i], s.B, s.K, s.N, s.ldb, 64, TC_BK))
            return cudaErrorInvalidValue;
    }
    const int work = P.total_work;
    int grid = work < num_sms ? work : num_sms;
    const cudaError_t e = launch_k(tc_tn_group_kernel, grid, TC_THREADS, TN_SMEM_BYTES, st, P);
    if (e != cudaSuccess) return e;
    int tiles = 0;
    for (int i = 0; i < n; ++i)
        if (P.p[i].splits > 1) tiles += P.p[i].num_m * P.p[i].num_n;
    if (tiles == 0) return cudaSuccess;
    return launch_k(tn_finish_kernel, tiles * TN_FINISH_SLABS, 256, 0, st, P);
}

}  // namespace grb
