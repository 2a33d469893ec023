// genrec_b200 - COBRA's generation and BeamFusion (genrec/models/cobra.py:531-760) on a prefix cache.
//
// The decoder runs once over each user's history (the prefill keeps every layer's QKV); each later codebook is one new token per
// beam, whose self-attention reads the history's K | V in place and the beam's own earlier tokens through an ancestry table:
//   cobra_attn_part_kernel     one CTA per (user, head, 128-key range of the history): the range's bf16 K / V loaded into shared
//                              memory once and scored against every query of the user (one warp per query, one key per lane);
//                              each query leaves its range's {acc[DH], max, sum} in the workspace
//   cobra_attn_merge_kernel    one warp per (query row, head): the ranges merged in range order, then the beam's suffix keys (its
//                              ancestors' tokens of earlier steps and its own), softmax in fp32, bf16 out
// The same two kernels serve the paged per-user pool (Cobra.new_pool): the history keys are addressed through KvPages (a null page
// table is the prefill's dense layout), a user has any number of queries (packed by offsets), and each query sees the keys 0 ..
// q_keys[r]-1.  The key ranges are fixed 128-position ranges of absolute position merged in order, so a query's result depends on
// its key limit and the keys' contents only, not on how the history was written or which users share the call.
//   cobra_kv_scatter_kernel    one warp per new decoder row: its K | V columns of the layer's QKV copied into the user's page row
//   cobra_beam_topk_kernel     one CTA per user: log_softmax(logits / temperature) per row plus the parent's score, and the K best
//                              of the user's K_in * V totals (beam_radix_topk of beam.cuh), best first, equal totals by the lower
//                              flat index; COBRA's parents are distinct and a parent's tokens are distinct, so nothing repeats and
//                              the step needs no dedup
//   cobra_dense_match_kernel   TMA + wgmma sweep of the catalog (tc_mainloop, K = D), one CTA per (row tile, item range) as
//                              sweep_range assigns them; each row's best (score, item) over the range
//   cobra_dense_merge_kernel   the ranges' winners in range order
// Every sum runs in a fixed order and no kernel uses atomics on values, so a user's results do not depend on the batch around it.
#pragma once
#include "attn_hstu_extend.cuh"
#include "beam.cuh"
#include "head_sweep.cuh"

namespace grb {

// ------------------------------------------------------------------------------------------------ beam attention
constexpr int CBA_CHUNK = 128;                  // history keys per CTA
constexpr int CBA_THREADS = 256;
constexpr int CBA_MAX_K = 1024;
constexpr int CBA_MAX_HIST = 8192;

struct CobraBeamAttnArgs {
    const bf16* q; int ldq;                     // [R, ldq]: query row r, head h at columns h DH ..
    const bf16* hk; const bf16* hv; int ldh;    // call row b's key j at hk[pg.row(u, j) ldh + h DH], u = users[b] (b without a list)
    KvPages pg;                                 // null page table: the prefill's QKV in place, page_size = its rows per user
    const int* users;                           // [B] page-table row of call row b, or null
    const int* hist_len;                        // [B]: call row b's keys are rows 0 .. hist_len[b]-1
    const int* q_off;                           // [B + 1]: call row b's queries are rows q_off[b] .. q_off[b+1]-1; null: b K .. b K + K-1
    const int* q_keys;                          // [R]: query r sees the keys 0 .. q_keys[r]-1 (<= hist_len of its row); null: hist_len[b]
    const bf16* sk; const bf16* sv; int lds;    // suffix step s, row r at sk[s step_stride + r lds]
    long long step_stride;
    const int* anc;                             // [R, S - 1]: the row of step s < S - 1 the beam descends from; step S - 1 is its own row
    int S;                                      // suffix keys per query (0: none)
    int B, K, R, H, splits;
    float scale;
    float* part;                                // [R H splits, DH + 2] {acc[DH], max, sum}
    bf16* out; int ldo;                         // [R, ldo]
};

template <int DH>
__global__ void __launch_bounds__(CBA_THREADS) cobra_attn_part_kernel(CobraBeamAttnArgs a) {
    pdl_wait();
    constexpr int LDS = DH + 2;                 // odd word stride: lane j reading row j is free of bank conflicts
    __shared__ bf16 sK[CBA_CHUNK * LDS];
    __shared__ bf16 sV[CBA_CHUNK * LDS];
    __shared__ float sQ[CBA_THREADS / 32][DH];
    const int sp = blockIdx.x % a.splits, bh = blockIdx.x / a.splits;
    const int h = bh % a.H, b = bh / a.H;
    const int j0 = sp * CBA_CHUNK;
    const int len = a.hist_len[b];
    if (j0 >= len) return;                      // the merge skips this range
    const int n = min(CBA_CHUNK, len - j0);
    const int u = a.users ? a.users[b] : b;
    for (int e = threadIdx.x; e < n * (DH / 2); e += CBA_THREADS) {
        const int j = e / (DH / 2), d2 = e - j * (DH / 2);
        const size_t g = a.pg.row(u, j0 + j) * a.ldh + h * DH + 2 * d2;
        *reinterpret_cast<uint32_t*>(&sK[j * LDS + 2 * d2]) = *reinterpret_cast<const uint32_t*>(a.hk + g);
        *reinterpret_cast<uint32_t*>(&sV[j * LDS + 2 * d2]) = *reinterpret_cast<const uint32_t*>(a.hv + g);
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int r0 = a.q_off ? a.q_off[b] : b * a.K;
    const int nq = a.q_off ? a.q_off[b + 1] - r0 : a.K;
    for (int k = warp; k < nq; k += CBA_THREADS / 32) {
        const int r = r0 + k;
        const int nk = a.q_keys ? min(n, a.q_keys[r] - j0) : n;     // the keys of this range the query sees
        if (nk <= 0) continue;                  // warp-uniform; the merge stops before this range
        const bf16* qr = a.q + (size_t)r * a.ldq + h * DH;
#pragma unroll
        for (int i = 0; i < DH / 32; ++i) sQ[warp][lane + 32 * i] = __bfloat162float(qr[lane + 32 * i]);
        __syncwarp();
        float m = -INFINITY, l = 0.f, acc[DH];
#pragma unroll
        for (int d = 0; d < DH; ++d) acc[d] = 0.f;
        for (int j = lane; j < nk; j += 32) {
            const uint32_t* kr = reinterpret_cast<const uint32_t*>(&sK[j * LDS]);
            float s = 0.f;
#pragma unroll
            for (int d2 = 0; d2 < DH / 2; ++d2) {
                const float2 kv = unpack_bf16(kr[d2]);
                s = __fmaf_rn(sQ[warp][2 * d2], kv.x, s);
                s = __fmaf_rn(sQ[warp][2 * d2 + 1], kv.y, s);
            }
            s *= a.scale;
            const uint32_t* vr = reinterpret_cast<const uint32_t*>(&sV[j * LDS]);
            float f = 1.f, e = 1.f;
            if (s > m) { f = __expf(m - s); m = s; }
            else e = __expf(s - m);
            l = l * f + e;
#pragma unroll
            for (int d2 = 0; d2 < DH / 2; ++d2) {
                const float2 vv = unpack_bf16(vr[d2]);
                acc[2 * d2] = acc[2 * d2] * f + e * vv.x;
                acc[2 * d2 + 1] = acc[2 * d2 + 1] * f + e * vv.y;
            }
        }
        float M = m;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) M = fmaxf(M, __shfl_xor_sync(0xffffffffu, M, o));
        const float f = l > 0.f ? __expf(m - M) : 0.f;
        l *= f;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) l += __shfl_xor_sync(0xffffffffu, l, o);
        float* dst = a.part + (((size_t)r * a.H + h) * a.splits + sp) * (DH + 2);
#pragma unroll
        for (int d = 0; d < DH; ++d) {
            float v = acc[d] * f;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
            if (lane == (d & 31)) dst[d] = v;
        }
        if (lane == 0) { dst[DH] = M; dst[DH + 1] = l; }
        __syncwarp();                           // sQ is rewritten by the next query
    }
}

template <int DH>
__global__ void __launch_bounds__(CBA_THREADS) cobra_attn_merge_kernel(CobraBeamAttnArgs a) {
    pdl_wait();
    constexpr int PER = DH / 32;                // dims of a lane: lane + 32 i
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long item = (long long)blockIdx.x * (CBA_THREADS / 32) + warp;       // (query row, head)
    if (item >= (long long)a.R * a.H) return;
    const int h = (int)(item % a.H);
    const int r = (int)(item / a.H);
    float q[PER], acc[PER];
    const bf16* qr = a.q + (size_t)r * a.ldq + h * DH;
#pragma unroll
    for (int i = 0; i < PER; ++i) { q[i] = __bfloat162float(qr[lane + 32 * i]); acc[i] = 0.f; }
    float M = -INFINITY, L = 0.f;
    const int len = a.q_keys ? a.q_keys[r] : a.hist_len[r / a.K];
    for (int sp = 0; sp < a.splits && sp * CBA_CHUNK < len; ++sp) {
        const float* src = a.part + (((size_t)r * a.H + h) * a.splits + sp) * (DH + 2);
        const float m = src[DH], l = src[DH + 1];
        const float Mn = fmaxf(M, m);
        const float fa = __expf(M - Mn), fb = __expf(m - Mn);
        L = L * fa + l * fb;
#pragma unroll
        for (int i = 0; i < PER; ++i) acc[i] = acc[i] * fa + src[lane + 32 * i] * fb;
        M = Mn;
    }
    for (int s = 0; s < a.S; ++s) {
        const int row = s < a.S - 1 ? a.anc[(size_t)r * (a.S - 1) + s] : r;
        const size_t g = (size_t)s * a.step_stride + (size_t)row * a.lds + h * DH;
        float part = 0.f;
#pragma unroll
        for (int i = 0; i < PER; ++i) part = __fmaf_rn(q[i], __bfloat162float(a.sk[g + lane + 32 * i]), part);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
        const float sc = __shfl_sync(0xffffffffu, part, 0) * a.scale;
        const float Mn = fmaxf(M, sc);
        const float fa = __expf(M - Mn), fb = __expf(sc - Mn);
        L = L * fa + fb;
#pragma unroll
        for (int i = 0; i < PER; ++i) acc[i] = acc[i] * fa + fb * __bfloat162float(a.sv[g + lane + 32 * i]);
        M = Mn;
    }
    bf16* o = a.out + (size_t)r * a.ldo + h * DH;
#pragma unroll
    for (int i = 0; i < PER; ++i) o[lane + 32 * i] = __float2bfloat16(__fdiv_rn(acc[i], L));
}

// Row r of a layer's QKV [R, ld_qkv] (K | V at columns D .. 3D-1) goes to row pg.row(row_user[r], row_pos[r]) of that layer's pages
// kv [pages page_size, 2D]; 16-byte copies, D a multiple of 8.
__global__ void __launch_bounds__(256) cobra_kv_scatter_kernel(const bf16* __restrict__ qkv, int ld_qkv, int R, int D, KvPages pg,
                                                               const int* __restrict__ row_user, const int* __restrict__ row_pos,
                                                               bf16* __restrict__ kv) {
    pdl_wait();
    const int r = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= R) return;
    const uint4* src = reinterpret_cast<const uint4*>(qkv + (size_t)r * ld_qkv + D);
    uint4* dst = reinterpret_cast<uint4*>(kv + pg.row(row_user[r], row_pos[r]) * (size_t)(2 * D));
    for (int i = lane; i < D / 4; i += 32) dst[i] = src[i];
}

// ------------------------------------------------------------------------------------------------ beam step
constexpr int CBT_MAX_CAND = BEAM_WIDE_MAX_CAND;

struct CobraTopkArgs {
    const float* logits;                        // [B K_in, V]
    const float* scores_in;                     // [B, K_in], or null (all zero)
    const int* anc_in;                          // [B K_in, S_in], or null when S_in = 0
    int B, K_in, V, K, S_in;
    float temperature;
    unsigned* mono;                             // [B, K_in V] workspace
    long long* tokens;                          // [B, K]
    float* scores;                              // [B, K]
    int* parents;                               // [B, K]
    int* anc_out;                               // [B K, S_in + 1], or null
};

// order-preserving key of a total, never 0; every NaN is larger than every number, as torch.topk orders them
GRB_DEVINL unsigned cobra_total_key(float t) { return t != t ? 0xffffffffu : beam_mono(t); }
GRB_DEVINL float cobra_key_total(unsigned m) {
    if (m == 0xffffffffu) return __int_as_float(0x7fffffff);
    return __uint_as_float((m & 0x80000000u) ? (m & 0x7fffffffu) : ~m);
}

__global__ void __launch_bounds__(BEAM_WIDE_THREADS) cobra_beam_topk_kernel(CobraTopkArgs a) {
    pdl_wait();
    __shared__ BeamRadixSmem s;
    __shared__ float s_max[CBA_MAX_K], s_lse[CBA_MAX_K];
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n = a.K_in * a.V;
    // log_softmax of each row of logits / temperature: {max, log sum exp(x - max)}, lane-strided sums reduced in a fixed order
    for (int p = warp; p < a.K_in; p += BEAM_WIDE_THREADS / 32) {
        const float* x = a.logits + ((size_t)b * a.K_in + p) * a.V;
        float m = -INFINITY;
        for (int v = lane; v < a.V; v += 32) m = fmaxf(m, __fdiv_rn(x[v], a.temperature));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
        float sum = 0.f;
        for (int v = lane; v < a.V; v += 32) sum += __expf(__fsub_rn(__fdiv_rn(x[v], a.temperature), m));
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (lane == 0) { s_max[p] = m; s_lse[p] = __logf(sum); }
    }
    __syncthreads();
    unsigned* mono = a.mono + (size_t)b * n;
    for (int f = tid; f < n; f += BEAM_WIDE_THREADS) {
        const int p = f / a.V;
        const float lp = __fsub_rn(__fsub_rn(__fdiv_rn(a.logits[(size_t)b * n + f], a.temperature), s_max[p]), s_lse[p]);
        const float t = a.scores_in ? __fadd_rn(a.scores_in[(size_t)b * a.K_in + p], lp) : lp;
        mono[f] = cobra_total_key(t);
    }
    __syncthreads();
    beam_radix_topk(mono, n, a.K, s);           // n >= K keys, none zero: K picks
    if (tid < a.K) {
        const unsigned long long key = s.key[tid];
        const int f = beam_key_flat(key), p = f / a.V;
        const size_t o = (size_t)b * a.K + tid;
        a.tokens[o] = f - p * a.V;
        a.scores[o] = cobra_key_total((unsigned)(key >> 32));
        a.parents[o] = p;
        if (a.anc_out) {
            const int pr = b * a.K_in + p;
            for (int j = 0; j < a.S_in; ++j) a.anc_out[o * (a.S_in + 1) + j] = a.anc_in[(size_t)pr * a.S_in + j];
            a.anc_out[o * (a.S_in + 1) + a.S_in] = pr;
        }
    }
}

// ------------------------------------------------------------------------------------------------ catalog match
constexpr int DMATCH_MAX_SPLITS = 256;

struct DenseMatchArgs {
    int R, N, splits, num_n, kblocks;
    float* cand_s;                              // [R, splits]
    int* cand_i;                                // [R, splits]
};

// Warp roles as tc_gemm_kernel; warp w of consumer warpgroup g owns rows 64 g + 16 w .. +15 of the tile and their running best.
__global__ void __launch_bounds__(TC_THREADS, 1)
    cobra_dense_match_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, DenseMatchArgs a) {
    extern __shared__ unsigned char dmatch_smem_raw[];
    unsigned char* base = dmatch_smem_raw + ((1024u - (smem_u32(dmatch_smem_raw) & 1023u)) & 1023u);
    unsigned char* sA = base;
    unsigned char* sB = base + TC_STAGES * TC_TILE_BYTES;
    float* sAcc = reinterpret_cast<float*>(base + 2 * TC_STAGES * TC_TILE_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(base + 2 * TC_STAGES * TC_TILE_BYTES + TC_ACC_BYTES);
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
    // ===================================================================== consumers: MMA + running best
    const int g = (warp >> 2) - 1;
    const int r0 = g * 64 + (warp & 3) * 16;
    float best_s = -INFINITY;                   // lane i < 16: row r0 + i
    int best_i = INT_MAX;
    int stage = 0;
    uint32_t phase = 0;
    float acc[64];
    for (int nt = t.n_begin; nt < t.n_end; ++nt) {
        tc_mainloop<0, 0, TC_STAGES>(acc, sA, sB, full_bar, empty_bar, 0, a.kblocks, g, stage, phase);
        wg_bar_sync(g);                          // this warpgroup's scan of the previous tile has read sAcc
        tc_acc_store(sAcc, acc, g);
        wg_bar_sync(g);
        const int n0 = nt * TC_BN;
#pragma unroll 1
        for (int i = 0; i < 16; ++i) {
            const int r = r0 + i;
            float ws = -INFINITY;
            int wid = INT_MAX;
#pragma unroll
            for (int q = 0; q < 4; ++q) {        // lane holds columns lane + 32 q
                const int c = 32 * q + lane;
                const float v = sAcc[r * TC_BN + (((c >> 2) ^ (r & 7)) << 2) + (c & 3)];
                if (n0 + c < a.N && topk_better(v, n0 + c, ws, wid)) { ws = v; wid = n0 + c; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const float s2 = __shfl_xor_sync(0xffffffffu, ws, o);
                const int i2 = __shfl_xor_sync(0xffffffffu, wid, o);
                if (topk_better(s2, i2, ws, wid)) { ws = s2; wid = i2; }
            }
            if (lane == i && topk_better(ws, wid, best_s, best_i)) { best_s = ws; best_i = wid; }
        }
    }
    const int row = m0 + r0 + lane;
    if (lane < 16 && row < a.R) {
        a.cand_s[(size_t)row * a.splits + t.split] = best_s;
        a.cand_i[(size_t)row * a.splits + t.split] = best_i;
    }
}

__global__ void __launch_bounds__(256) cobra_dense_merge_kernel(const float* cand_s, const int* cand_i, int R, int splits, float* best,
                                                                long long* item) {
    pdl_wait();
    const int row = blockIdx.x * 256 + threadIdx.x;
    if (row >= R) return;
    float bs = -INFINITY;
    int bi = INT_MAX;
    for (int s = 0; s < splits; ++s) {
        const float v = cand_s[(size_t)row * splits + s];
        const int id = cand_i[(size_t)row * splits + s];
        if (topk_better(v, id, bs, bi)) { bs = v; bi = id; }
    }
    best[row] = bs;
    item[row] = bi;
}

}  // namespace grb
