// genrec_b200 - sampled-softmax head on wgmma: every token is scored against its target and against N negatives shared by the
// whole call, with a logQ correction; loss, d(loss)/d(x) and d(loss)/d(table) in time that does not depend on the catalog size.
// D = 64 or 128.  No [tokens, negatives] tensor is written.
//
//   sce_gather_kernel   Es [Npad, D] bf16 = the table rows of the negatives (Npad = N rounded up to the 64-class tile), the
//                       per-class bias -log_q[s_j] (-inf for padding classes and ids outside 1 .. C-1) and the checked ids.
//   sce_target_kernel   z_tgt[t] = h_t . E[y_t] - log_q[y_t]: one warp per token, a gather-dot.
//   sce_rows_kernel     row-stationary, one CTA per 128-token tile: the token tile stays in shared
//                       memory and Es streams through a TMA ring twice.  Sweep 1: S = H Es^T + bias, accidental hits (s_j == y_t)
//                       masked, online maximum / exponent sum starting from the target column -> per-row loss and log2-domain
//                       shift.  Sweep 2: S again, G in registers -> bf16 A operand of dH += G Es; the target's own term
//                       g_tgt E[y_t] is added in the epilogue.  N is small, so a row tile's sweep is not cut into segments: one
//                       unit per row tile, 200 units on 132 SMs at 128 x 200 tokens (two rounds where 1.52 would do).
//   sce_table_kernel    class-stationary: CTA (class tile, token range k) sums G^T H over its
//                       token range into part[k][Npad][D]; the ranges are added in index order by the scatter.
//   sce_scatter_kernel  dtable[id] += for the negatives and the targets.  CTA p owns the table rows id % P == p: it walks the
//                       negatives, then the tokens, in index order, keeps the ones it owns, and the first occurrence of an id sums
//                       all its occurrences in that order.  One writer per table row, no sort, no order-dependent atomics.
// The row and table kernels are built from the tile steps of tc_ce.cuh (ce_cta_init, ce_tile_load / ce_ring_load, ce_lane,
// ce_softmax_step, ce_row_finish, ce_table_cols, ce_wg_handover), so the ring, the barriers, the softmax arithmetic and the bf16
// rounding of G for the two wgmma products are the full head's by construction; g_tgt stays fp32.
#pragma once
#include "tc_ce.cuh"

namespace grb {

constexpr int SCE_MAX_N = 8192;
constexpr int SCE_SCATTER_THREADS = 512;
constexpr int SCE_WINDOW = 8 * SCE_SCATTER_THREADS;   // items (negatives, then tokens) a scatter CTA filters per round

struct SceArgs {
    const long long* tg;        // [T] targets (0 = ignored)
    const long long* neg;       // [N] negatives
    const float* log_q;         // [C] or null
    const bf16* table;          // [C, D]
    const bf16* xf;             // [T, D] bf16(LayerNorm(x))
    const float* inv_count;     // device scalar: 1 / #(targets != 0)
    int T, C, N, Npad, D;
    bf16* Es;                   // [Npad, D]
    float* bias;                // [Npad]
    int* sid;                   // [Npad] the negative's id, -1 when it is padding or outside 1 .. C-1
    float* ztgt;                // [T] corrected target score
    float* shift;               // [T] log2-domain lse
    float* row_loss;            // [T]
    float* gtgt;                // [T] (p_tgt - 1) / count, formed as -(sum of the negatives' G)
    float* dxf;                 // [T, D] d loss / d h (nullable: loss only)
    float* part;                // [ks][Npad][D] per-token-range sums of G^T H
    int ks;
    float* dtable;              // [C, D] +=
};

// a target the kernels act on: inside 1 .. C-1, else 0 (ignored)
GRB_DEVINL int sce_target(const long long* tg, int t, int T, int C) {
    if (t >= T) return 0;
    const long long y = tg[t];
    return y >= 1 && y < C ? (int)y : 0;
}

__global__ void __launch_bounds__(256) sce_gather_kernel(SceArgs a) {
    pdl_wait();
    const int j = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (j >= a.Npad) return;
    const long long id = j < a.N ? a.neg[j] : 0;
    const bool ok = id >= 1 && id < a.C;
    for (int c = 4 * lane; c < a.D; c += 128) {
        uint2 v = make_uint2(0u, 0u);
        if (ok) v = *reinterpret_cast<const uint2*>(a.table + (size_t)id * a.D + c);
        *reinterpret_cast<uint2*>(a.Es + (size_t)j * a.D + c) = v;
    }
    if (lane == 0) {
        a.bias[j] = ok ? (a.log_q ? -a.log_q[id] : 0.f) : -INFINITY;
        a.sid[j] = ok ? (int)id : -1;
    }
}

__global__ void __launch_bounds__(256) sce_target_kernel(SceArgs a) {
    pdl_wait();
    const int t = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (t >= a.T) return;
    const int y = sce_target(a.tg, t, a.T, a.C);
    float s = 0.f;
    if (y != 0)
        for (int c = 4 * lane; c < a.D; c += 128) {
            const uint2 h = *reinterpret_cast<const uint2*>(a.xf + (size_t)t * a.D + c);
            const uint2 e = *reinterpret_cast<const uint2*>(a.table + (size_t)y * a.D + c);
            const float2 h0 = unpack_bf16(h.x), h1 = unpack_bf16(h.y), e0 = unpack_bf16(e.x), e1 = unpack_bf16(e.y);
            s += h0.x * e0.x + h0.y * e0.y + h1.x * e1.x + h1.y * e1.y;
        }
    s = warp_sum(s);
    if (lane == 0) a.ztgt[t] = y != 0 ? s - (a.log_q ? a.log_q[y] : 0.f) : 0.f;
}

template <int D>
constexpr int sce_rows_smem(int Npad) { return CeSmem<D>::ROWS_BYTES + 8 * Npad; }

template <int D>
__global__ void __launch_bounds__(CE_THREADS, 1)
    sce_rows_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmE, SceArgs a) {
    using SM = CeSmem<D>;
    extern __shared__ unsigned char ce_smem_raw[];
    const CeCta cta = ce_cta_init<D>(ce_smem_raw, SM::ROW_TILE, 2, &tmX, &tmE);
    float* sBias = reinterpret_cast<float*>(cta.tail);
    int* sSid = reinterpret_cast<int*>(sBias + a.Npad);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp >= 1 && warp < 4) return;            // warp 0 produces (lane 0 issues the loads), warps 4..11 consume
    const int ntile = a.Npad / 64, row0 = blockIdx.x * 128;
    const int sweeps = a.dxf ? 2 : 1;
    int stage = 0;
    uint32_t phase = 0;
    if (warp == 0) {
        if (lane == 0) {
            ce_tile_load<D, 128>(cta, &tmX, row0);
            for (int n = 0; n < sweeps * ntile; ++n) {
                ce_ring_load<D>(cta, &tmE, n % ntile * 64, stage, phase ^ 1);
                if (++stage == CE_STAGES) { stage = 0; phase ^= 1; }
            }
        }
        return;
    }
    const CeLane l = ce_lane();                    // consumer warpgroup g: tile rows 64 g .. 64 g + 63
    const int q = l.q;
    for (int i = threadIdx.x - 128; i < a.Npad; i += 256) {
        sBias[i] = a.bias[i];
        sSid[i] = a.sid[i];
    }
    int row[2], tgt[2];
    float ic[2], zt[2];
    const float inv = *a.inv_count;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        row[i] = l.row(row0 + 64 * l.g, i);
        tgt[i] = sce_target(a.tg, row[i], a.T, a.C);
        ic[i] = tgt[i] != 0 ? inv : 0.f;
        zt[i] = tgt[i] != 0 ? a.ztgt[row[i]] : 0.f;
    }
    ce_bar(2, 256);
    mbar_wait(cta.sfull, 0);
    const uint32_t xa = smem_u32(cta.stat) + l.g * 8192;
    // the softmax starts from the target column (the quad's lane 0 carries its exponent); an accidental hit never enters it
    float m[2] = {zt[0], zt[1]}, s[2] = {q == 0 ? 1.f : 0.f, q == 0 ? 1.f : 0.f};
    for (int j = 0; j < ntile; ++j) {
        mbar_wait(&cta.full[stage], phase);
        float S[32];
        ce_scores<D>(S, xa, 16384, smem_u32(cta.ring + stage * SM::CLS_TILE));
        if (l.leader) mbar_arrive(&cta.empty[stage]);
        if (++stage == CE_STAGES) { stage = 0; phase ^= 1; }
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            const int col = j * 64 + 8 * jj + 2 * q;
            const float2 b = *reinterpret_cast<const float2*>(sBias + col);
            const int2 id = *reinterpret_cast<const int2*>(sSid + col);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                S[jj * 4 + i * 2] = id.x == tgt[i] ? -INFINITY : S[jj * 4 + i * 2] + b.x;
                S[jj * 4 + i * 2 + 1] = id.y == tgt[i] ? -INFINITY : S[jj * 4 + i * 2 + 1] + b.y;
            }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) ce_softmax_step(S, i, m[i], s[i]);
    }
    float shift[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        float lse;
        shift[i] = ce_row_finish(m[i], s[i], lse);
        if (q == 0 && row[i] < a.T) {
            a.row_loss[row[i]] = tgt[i] != 0 ? (lse - zt[i]) * ic[i] : 0.f;
            a.shift[row[i]] = shift[i];
        }
    }
    if (!a.dxf) return;
    // rows past T and ignored rows: zero weights, so their G is 0 whatever the shift
    float dx[D / 2];
#pragma unroll
    for (int kk = 0; kk < D / 2; ++kk) dx[kk] = 0.f;
    float gsum[2] = {0.f, 0.f};                    // sum_j G of the row: g_tgt = (p_tgt - 1) / count = -gsum, without the cancellation
    for (int j = 0; j < ntile; ++j) {
        mbar_wait(&cta.full[stage], phase);
        float S[32];
        const uint32_t e_addr = smem_u32(cta.ring + stage * SM::CLS_TILE);
        ce_scores<D>(S, xa, 16384, e_addr);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
            const int col = j * 64 + 8 * jj + 2 * q;
            const float2 b = *reinterpret_cast<const float2*>(sBias + col);
            const int2 id = *reinterpret_cast<const int2*>(sSid + col);
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                float& v0 = S[jj * 4 + i * 2];
                float& v1 = S[jj * 4 + i * 2 + 1];
                v0 = id.x == tgt[i] ? 0.f : ex2_fast((v0 + b.x) * CE_L2E - shift[i]) * ic[i];
                v1 = id.y == tgt[i] ? 0.f : ex2_fast((v1 + b.y) * CE_L2E - shift[i]) * ic[i];
                gsum[i] += v0 + v1;
            }
        }
        ce_accumulate<D>(dx, S, e_addr);
        if (l.leader) mbar_arrive(&cta.empty[stage]);
        if (++stage == CE_STAGES) { stage = 0; phase ^= 1; }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        gsum[i] += __shfl_xor_sync(0xffffffffu, gsum[i], 1);
        gsum[i] += __shfl_xor_sync(0xffffffffu, gsum[i], 2);
        if (row[i] >= a.T) continue;
        const float gt = -gsum[i];
        if (q == 0) a.gtgt[row[i]] = gt;
        const bf16* er = a.table + (size_t)tgt[i] * D;      // row 0 when the token is ignored: gt is 0 then
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj) {
            const float2 e = unpack_bf16(*reinterpret_cast<const uint32_t*>(er + 8 * jj + 2 * q));
            *reinterpret_cast<float2*>(a.dxf + (size_t)row[i] * D + 8 * jj + 2 * q) =
                make_float2(dx[jj * 4 + i * 2] + gt * e.x, dx[jj * 4 + i * 2 + 1] + gt * e.y);
        }
    }
}

// CTA (ct, k): class tile ct of Es, token tiles [k ntt / ks, (k + 1) ntt / ks); consumer warpgroup g takes the tiles tt = g (mod 2)
template <int D>
__global__ void __launch_bounds__(CE_THREADS, 1)
    sce_table_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmE, SceArgs a) {
    using SM = CeSmem<D>;
    extern __shared__ unsigned char ce_smem_raw[];
    const CeCta cta = ce_cta_init<D>(ce_smem_raw, SM::CLS_TILE, 1, &tmX, &tmE);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp >= 1 && warp < 4) return;
    const int ntt = (a.T + 63) / 64, ct = blockIdx.x, k = blockIdx.y, cls0 = ct * 64;
    const int t0 = (int)((long long)k * ntt / a.ks), t1 = (int)((long long)(k + 1) * ntt / a.ks);
    if (warp == 0) {
        if (lane == 0) {
            ce_tile_load<D, 64>(cta, &tmE, cls0);
            for (int tt = t0; tt < t1; ++tt) {
                const int p = tt - t0;
                ce_ring_load<D>(cta, &tmX, tt * 64, p % CE_STAGES, ((p / CE_STAGES) & 1) ^ 1);
            }
        }
        return;
    }
    const CeLane l = ce_lane();
    const int q = l.q;
    int cid[2];
    float cb[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        cid[i] = a.sid[l.row(cls0, i)];
        cb[i] = a.bias[l.row(cls0, i)];
    }
    const float inv = *a.inv_count;
    float acc[D / 2];
#pragma unroll
    for (int kk = 0; kk < D / 2; ++kk) acc[kk] = 0.f;
    mbar_wait(cta.sfull, 0);
    const uint32_t ea = smem_u32(cta.stat);
    for (int tt = t0 + ((t0 ^ l.g) & 1); tt < t1; tt += 2) {
        const int p = tt - t0;
        const int stage = p % CE_STAGES;
        CeCols col;
        ce_table_cols(col, l, tt, a.T, a.shift, inv, [&](int t) { return sce_target(a.tg, t, a.T, a.C); });
        mbar_wait(&cta.full[stage], (p / CE_STAGES) & 1);
        const uint32_t x_addr = smem_u32(cta.ring + stage * SM::CLS_TILE);
        float S[32];
        ce_scores<D>(S, ea, 8192, x_addr);     // S^T: rows = the 64 classes, columns = 64 tokens
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    float& v = S[jj * 4 + i * 2 + c];
                    const int kq = jj * 2 + c;
                    v = cid[i] == col.tg[kq] ? 0.f : ex2_fast((v + cb[i]) * CE_L2E - col.sh[kq]) * col.icc[kq];
                }
        ce_accumulate<D>(acc, S, x_addr);
        if (l.leader) mbar_arrive(&cta.empty[stage]);
    }
    ce_wg_handover<D>(cta, l, acc);
    if (l.g == 0) {
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int kk = jj * 4 + i * 2;
                *reinterpret_cast<float2*>(a.part + ((size_t)k * a.Npad + l.row(cls0, i)) * D + 8 * jj + 2 * q) =
                    make_float2(acc[kk] + ce_wg_peer(cta, kk), acc[kk + 1] + ce_wg_peer(cta, kk + 1));
            }
    }
}

// Items 0 .. N-1 are the negatives, N .. N+T-1 the tokens.  CTA p keeps, in item order, the items whose id is in 1 .. C-1 and
// id % gridDim.x == p; the first occurrence of an id in a round sums every occurrence of the round in item order (a negative
// brings the sum of its token-range partials in range order, a token g_tgt h_t) and adds the sum to the table row once.  Rounds
// follow one another on the same CTA, so a row's additions have one order whatever the timing.
__global__ void __launch_bounds__(SCE_SCATTER_THREADS) sce_scatter_kernel(SceArgs a) {
    pdl_wait();
    __shared__ int l_item[SCE_WINDOW], l_id[SCE_WINDOW], wcnt[SCE_SCATTER_THREADS / 32];
    constexpr int NW = SCE_SCATTER_THREADS / 32, PER = SCE_WINDOW / SCE_SCATTER_THREADS;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int items = a.N + a.T, P = gridDim.x, me = blockIdx.x;
    const int col = 4 * lane;      // D = 64: lanes 0..15 carry the row, D = 128: all 32
    for (int w0 = 0; w0 < items; w0 += SCE_WINDOW) {
        int ids[PER];
        unsigned bal[PER];
        int cnt = 0;
#pragma unroll
        for (int c = 0; c < PER; ++c) {
            const int it = w0 + (warp * PER + c) * 32 + lane;
            long long id = 0;
            if (it < a.N) id = a.neg[it];
            else if (it < items) id = a.tg[it - a.N];
            const bool mine = id >= 1 && id < a.C && (int)(id % P) == me;
            ids[c] = (int)id;
            bal[c] = __ballot_sync(0xffffffffu, mine);
            cnt += __popc(bal[c]);
        }
        if (lane == 0) wcnt[warp] = cnt;
        __syncthreads();
        int at = 0, n = 0;
        for (int i = 0; i < NW; ++i) {
            if (i < warp) at += wcnt[i];
            n += wcnt[i];
        }
#pragma unroll
        for (int c = 0; c < PER; ++c) {
            if (bal[c] >> lane & 1u) {
                const int pos = at + __popc(bal[c] & ((1u << lane) - 1u));
                l_item[pos] = w0 + (warp * PER + c) * 32 + lane;
                l_id[pos] = ids[c];
            }
            at += __popc(bal[c]);
        }
        __syncthreads();
        for (int e = warp; e < n; e += NW) {
            const int id = l_id[e];
            bool seen = false;
            for (int e0 = 0; e0 < e && !seen; e0 += 32) seen = __any_sync(0xffffffffu, e0 + lane < e && l_id[e0 + lane] == id);
            if (seen) continue;
            float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
            for (int e0 = e & ~31; e0 < n; e0 += 32) {
                const int ee = e0 + lane;
                unsigned same = __ballot_sync(0xffffffffu, ee >= e && ee < n && l_id[ee] == id);
                while (same) {
                    const int it = l_item[e0 + __ffs(same) - 1];
                    same &= same - 1;
                    if (col >= a.D) continue;
                    if (it < a.N) {
                        for (int k = 0; k < a.ks; ++k) {
                            const float4 v = *reinterpret_cast<const float4*>(a.part + ((size_t)k * a.Npad + it) * a.D + col);
                            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
                        }
                    } else {
                        const int t = it - a.N;
                        const float gt = a.gtgt[t];
                        const uint2 h = *reinterpret_cast<const uint2*>(a.xf + (size_t)t * a.D + col);
                        const float2 h0 = unpack_bf16(h.x), h1 = unpack_bf16(h.y);
                        acc.x += gt * h0.x; acc.y += gt * h0.y; acc.z += gt * h1.x; acc.w += gt * h1.y;
                    }
                }
            }
            if (col < a.D) red_add_v4(a.dtable + (size_t)id * a.D + col, acc.x, acc.y, acc.z, acc.w);   // one add per row and round
        }
        __syncthreads();
    }
}

// token ranges of the table pass: class tiles x ranges fill the SMs once, never more ranges than 64-token tiles
inline int sce_table_splits(int T, int Npad, int sms) {
    const int nc = Npad / 64, ntt = (T + 63) / 64;
    int ks = sms / nc;
    ks = ks < ntt ? ks : ntt;
    return ks < 1 ? 1 : ks;
}

// the whole sampled head after the LayerNorm forward and the target count: loss per row, dxf, dtable +=
template <int D>
inline cudaError_t launch_sampled_ce(const SceArgs& a, int sms, cudaStream_t st) {
    CUtensorMap tmX128, tmX64, tmE;
    if (!make_tmap_bf16(&tmX128, a.xf, a.T, D, D, 64, 128) || !make_tmap_bf16(&tmX64, a.xf, a.T, D, D, 64, 64) ||
        !make_tmap_bf16(&tmE, a.Es, a.Npad, D, D, 64, 64))
        return cudaErrorInvalidValue;
    // the row kernel asks for its largest size once, so no later call with more negatives has to raise the attribute
    cudaError_t e = set_max_smem(sce_rows_kernel<D>, sce_rows_smem<D>(SCE_MAX_N));
    if (e == cudaSuccess) e = launch_k(sce_gather_kernel, (a.Npad + 7) / 8, 256, 0, st, a);
    if (e == cudaSuccess) e = launch_k(sce_target_kernel, (a.T + 7) / 8, 256, 0, st, a);
    if (e == cudaSuccess) e = launch_k(sce_rows_kernel<D>, (a.T + 127) / 128, CE_THREADS, sce_rows_smem<D>(a.Npad), st, tmX128, tmE, a);
    if (e != cudaSuccess || !a.dxf) return e;
    e = launch_k(sce_table_kernel<D>, dim3(a.Npad / 64, a.ks), CE_THREADS, CeSmem<D>::TABLE_BYTES, st, tmX64, tmE, a);
    if (e == cudaSuccess) e = launch_k(sce_scatter_kernel, 2 * sms, SCE_SCATTER_THREADS, 0, st, a);
    return e;
}

}  // namespace grb
