// genrec_b200 - SASRec causal softmax attention (reference: genrec/models/sasrec.py:206-240), flash-style, mma.sync path.
//
//   S = (Q K^T) * dh^-1/2 ; masked where j > i or key j is padding ; A = softmax_j(S) * qmask[i] ; out = drop(A) V
// A padded query row has qmask = 0, so its output is exactly 0 (the reference's "uniform softmax over -1e9" never
// survives the post-softmax query mask, sasrec.py:232-233); a non-padded query always sees its own key.
// Shares tile/fragment helpers with attn_hstu.cuh.
//
// Packed (jagged) batches: with SasAttnArgs::offsets set, sequence b is token rows offsets[b] .. offsets[b+1]-1 of T, clamped to
// [0, T) and to L = the longest length the grid covers (seq_span).  A query tile past a sequence's end exits at once.  lse is then
// per token, [H, T].  Under dropout the mask of a packed batch is keyed by the query's TOKEN ROW and the head, and by the key's
// index within its sequence: row key (tok0 + i) * H + h, column j; the padded layout keeps row key (b H + h) L + i, column j.
// The kernels write only sequence rows: the caller zeroes the idle rows [0, offsets[0]) and [offsets[B], T) of O and dQ | dK | dV.
// JAGGED is a template parameter, so the padded instantiations compile to the code they had before packed batches existed.
#pragma once
#include "attn_hstu.cuh"

namespace grb {

struct SasAttnArgs {
    const bf16* q; const bf16* k; const bf16* v; int ld;  // [T, D] each
    const uint8_t* pad;                                   // [B, L] (packed: [T]) 1 = padding (mask == 0)
    int B, L, H;
    float scale;
    Dropout drop;
    bf16* out; float* lse;                                // out [T, D] ; lse [B, H, L]
    const bf16* d_out;                                    // [T, D]
    bf16* dq; bf16* dk; bf16* dv;                         // [T, D]
    const long long* offsets;                             // packed batch: [B+1] (null: sequence b is rows b*L .. b*L+L-1)
    int T;                                                // packed batch: token rows
};

// lse slot and dropout row key of query i of sequence b (first row tok0, L rows), head h
template <bool JAGGED>
GRB_DEVINL size_t sas_lse_at(const SasAttnArgs& a, int b, int h, long long tok0, int L, int i) {
    return JAGGED ? (size_t)h * a.T + (size_t)(tok0 + i) : ((size_t)b * a.H + h) * L + i;
}
template <bool JAGGED>
GRB_DEVINL uint32_t sas_drop_row(const SasAttnArgs& a, int b, int h, long long tok0, int L, int i) {
    return JAGGED ? ((uint32_t)tok0 + (uint32_t)i) * (uint32_t)a.H + (uint32_t)h : (uint32_t)((b * a.H + h) * L + i);
}

template <int DH>
struct SasSmem {
    static constexpr int LD = DH + 8;
    bf16 tile[5][ATT_BLK * LD];
    float lse_tile[ATT_BLK];
    float dsum_tile[ATT_BLK];
    uint8_t pad_tile[ATT_BLK];
};

GRB_DEVINL float quad_max(float v) {
    v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
    return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
GRB_DEVINL float quad_sum(float v) {
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// tile roles: 0 = Q, 1 = K, 2 = V
template <int DH, bool JAGGED>
__global__ void __launch_bounds__(ATT_THREADS) sas_attn_fwd_kernel(SasAttnArgs a) {
    pdl_wait();
    a.drop.resolve();
    extern __shared__ __align__(16) unsigned char att_smem_raw[];
    SasSmem<DH>& sm = *reinterpret_cast<SasSmem<DH>*>(att_smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int q0 = qt * ATT_BLK;
    long long tok0;
    int L;
    seq_span<JAGGED>(a.offsets, a.T, a.L, b, tok0, L);
    if (JAGGED && q0 >= L) return;   // query tile past the end of a packed sequence

    att_load_tile<DH>(sm.tile[0], a.q + (size_t)tok0 * a.ld + h * DH, a.ld, 0, q0, L, 0, tid);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    uint32_t qf[DH / 16][4];
    att_load_afrag<DH>(qf, sm.tile[0], warp * 16, lane);
    const int i0 = q0 + warp * 16 + g, i1 = i0 + 8;
    const bool qok0 = i0 < L && a.pad[tok0 + i0] == 0, qok1 = i1 < L && a.pad[tok0 + i1] == 0;

    float o[DH / 8][4];
#pragma unroll
    for (int n = 0; n < DH / 8; ++n)
#pragma unroll
        for (int r = 0; r < 4; ++r) o[n][r] = 0.f;
    float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;

    for (int kt = 0; kt <= qt; ++kt) {
        const int k0 = kt * ATT_BLK;
        __syncthreads();
        att_load_tile<DH>(sm.tile[1], a.k + (size_t)tok0 * a.ld + h * DH, a.ld, 0, k0, L, 0, tid);
        att_load_tile<DH>(sm.tile[2], a.v + (size_t)tok0 * a.ld + h * DH, a.ld, 0, k0, L, 0, tid);
        cp_async_commit();
        if (tid < ATT_BLK) sm.pad_tile[tid] = (k0 + tid < L) ? a.pad[tok0 + k0 + tid] : 1;
        cp_async_wait<0>();
        __syncthreads();

        float s[8][4];
#pragma unroll
        for (int n = 0; n < 8; ++n)
#pragma unroll
            for (int r = 0; r < 4; ++r) s[n][r] = 0.f;
        att_mma_nt<DH>(s, qf, sm.tile[1], lane);
        float tm0 = -INFINITY, tm1 = -INFINITY;
#pragma unroll
        for (int n = 0; n < 8; ++n)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int jl = n * 8 + 2 * t + (r & 1), j = k0 + jl;
                const int i = (r < 2) ? i0 : i1;
                const bool valid = (j <= i) && ((r < 2) ? qok0 : qok1) && sm.pad_tile[jl] == 0;
                float v = valid ? s[n][r] * a.scale : -INFINITY;
                s[n][r] = v;
                if (r < 2) tm0 = fmaxf(tm0, v); else tm1 = fmaxf(tm1, v);
            }
        tm0 = quad_max(tm0); tm1 = quad_max(tm1);
        const float nm0 = fmaxf(m0, tm0), nm1 = fmaxf(m1, tm1);
        const float al0 = (nm0 == -INFINITY) ? 1.f : __expf(m0 - nm0), al1 = (nm1 == -INFINITY) ? 1.f : __expf(m1 - nm1);
        float rs0 = 0.f, rs1 = 0.f;
#pragma unroll
        for (int n = 0; n < 8; ++n)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const float nm = (r < 2) ? nm0 : nm1;
                float p = (s[n][r] == -INFINITY) ? 0.f : __expf(s[n][r] - nm);
                if (r < 2) rs0 += p; else rs1 += p;
                if (a.drop.thresh) {
                    const int jl = n * 8 + 2 * t + (r & 1);
                    const int i = (r < 2) ? i0 : i1;
                    p = a.drop.apply(p, sas_drop_row<JAGGED>(a, b, h, tok0, L, i), (uint32_t)(k0 + jl));
                }
                s[n][r] = p;
            }
        l0 = l0 * al0 + quad_sum(rs0);
        l1 = l1 * al1 + quad_sum(rs1);
        m0 = nm0; m1 = nm1;
#pragma unroll
        for (int n = 0; n < DH / 8; ++n) {
            o[n][0] *= al0; o[n][1] *= al0; o[n][2] *= al1; o[n][3] *= al1;
        }
        uint32_t pf[4][4];
        att_pack_p(pf, s);
        att_mma_nn<DH>(o, pf, sm.tile[2], lane);
    }
    const float inv0 = l0 > 0.f ? 1.f / l0 : 0.f, inv1 = l1 > 0.f ? 1.f / l1 : 0.f;
#pragma unroll
    for (int n = 0; n < DH / 8; ++n) {
        int col = h * DH + n * 8 + 2 * t;
        if (i0 < L) *reinterpret_cast<uint32_t*>(a.out + (size_t)(tok0 + i0) * a.ld + col) = pack_bf16(o[n][0] * inv0, o[n][1] * inv0);
        if (i1 < L) *reinterpret_cast<uint32_t*>(a.out + (size_t)(tok0 + i1) * a.ld + col) = pack_bf16(o[n][2] * inv1, o[n][3] * inv1);
    }
    if (t == 0) {
        if (i0 < L) a.lse[sas_lse_at<JAGGED>(a, b, h, tok0, L, i0)] = l0 > 0.f ? m0 + logf(l0) : 0.f;
        if (i1 < L) a.lse[sas_lse_at<JAGGED>(a, b, h, tok0, L, i1)] = l1 > 0.f ? m1 + logf(l1) : 0.f;
    }
}

// rowsum(dO * O) for the 64 rows of (tile_do, tile_o) -> dsum[64] ; 2 threads per row
template <int DH>
GRB_DEVINL void sas_rowdot(float* dsum, const bf16* tdo, const bf16* to, int tid) {
    constexpr int LD = DH + 8;
    const int r = tid >> 1, half = tid & 1;
    float s = 0.f;
#pragma unroll
    for (int c = 0; c < DH / 2; ++c) {
        int cc = half * (DH / 2) + c;
        s += __bfloat162float(tdo[r * LD + cc]) * __bfloat162float(to[r * LD + cc]);
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    if (half == 0) dsum[r] = s;
}

// backward dQ: tile roles 0 = Q, 1 = K, 2 = V, 3 = dO, 4 = O
template <int DH, bool JAGGED>
__global__ void __launch_bounds__(ATT_THREADS) sas_attn_bwd_dq_kernel(SasAttnArgs a) {
    pdl_wait();
    a.drop.resolve();
    extern __shared__ __align__(16) unsigned char att_smem_raw[];
    SasSmem<DH>& sm = *reinterpret_cast<SasSmem<DH>*>(att_smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int q0 = qt * ATT_BLK;
    long long tok0;
    int L;
    seq_span<JAGGED>(a.offsets, a.T, a.L, b, tok0, L);
    if (JAGGED && q0 >= L) return;   // query tile past the end of a packed sequence

    att_load_tile<DH>(sm.tile[0], a.q + (size_t)tok0 * a.ld + h * DH, a.ld, 0, q0, L, 0, tid);
    att_load_tile<DH>(sm.tile[3], a.d_out + (size_t)tok0 * a.ld + h * DH, a.ld, 0, q0, L, 0, tid);
    att_load_tile<DH>(sm.tile[4], a.out + (size_t)tok0 * a.ld + h * DH, a.ld, 0, q0, L, 0, tid);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    sas_rowdot<DH>(sm.dsum_tile, sm.tile[3], sm.tile[4], tid);
    if (tid < ATT_BLK) sm.lse_tile[tid] = (q0 + tid < L) ? (JAGGED ? a.lse[(size_t)h * a.T + (size_t)(tok0 + q0 + tid)] : a.lse[((size_t)b * a.H + h) * L + q0 + tid]) : 0.f;
    __syncthreads();
    uint32_t qf[DH / 16][4], dof[DH / 16][4];
    att_load_afrag<DH>(qf, sm.tile[0], warp * 16, lane);
    att_load_afrag<DH>(dof, sm.tile[3], warp * 16, lane);
    const int i0 = q0 + warp * 16 + g, i1 = i0 + 8;
    const bool qok0 = i0 < L && a.pad[tok0 + i0] == 0, qok1 = i1 < L && a.pad[tok0 + i1] == 0;
    const float lse0 = sm.lse_tile[warp * 16 + g], lse1 = sm.lse_tile[warp * 16 + g + 8];
    const float ds0 = sm.dsum_tile[warp * 16 + g], ds1 = sm.dsum_tile[warp * 16 + g + 8];
    float dq[DH / 8][4];
#pragma unroll
    for (int n = 0; n < DH / 8; ++n)
#pragma unroll
        for (int r = 0; r < 4; ++r) dq[n][r] = 0.f;

    for (int kt = 0; kt <= qt; ++kt) {
        const int k0 = kt * ATT_BLK;
        __syncthreads();
        att_load_tile<DH>(sm.tile[1], a.k + (size_t)tok0 * a.ld + h * DH, a.ld, 0, k0, L, 0, tid);
        att_load_tile<DH>(sm.tile[2], a.v + (size_t)tok0 * a.ld + h * DH, a.ld, 0, k0, L, 0, tid);
        cp_async_commit();
        if (tid < ATT_BLK) sm.pad_tile[tid] = (k0 + tid < L) ? a.pad[tok0 + k0 + tid] : 1;
        cp_async_wait<0>();
        __syncthreads();
        float s[8][4], da[8][4];
#pragma unroll
        for (int n = 0; n < 8; ++n)
#pragma unroll
            for (int r = 0; r < 4; ++r) s[n][r] = 0.f, da[n][r] = 0.f;
        att_mma_nt<DH>(s, qf, sm.tile[1], lane);
        att_mma_nt<DH>(da, dof, sm.tile[2], lane);
#pragma unroll
        for (int n = 0; n < 8; ++n)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int jl = n * 8 + 2 * t + (r & 1), j = k0 + jl;
                const int i = (r < 2) ? i0 : i1;
                const bool valid = (j <= i) && ((r < 2) ? qok0 : qok1) && sm.pad_tile[jl] == 0;
                float dsv = 0.f;
                if (valid) {
                    float p = __expf(s[n][r] * a.scale - ((r < 2) ? lse0 : lse1));
                    float dA = a.drop.apply(da[n][r], sas_drop_row<JAGGED>(a, b, h, tok0, L, i), (uint32_t)j);
                    dsv = p * (dA - ((r < 2) ? ds0 : ds1)) * a.scale;
                }
                s[n][r] = dsv;
            }
        uint32_t pf[4][4];
        att_pack_p(pf, s);
        att_mma_nn<DH>(dq, pf, sm.tile[1], lane);
    }
#pragma unroll
    for (int n = 0; n < DH / 8; ++n) {
        int col = h * DH + n * 8 + 2 * t;
        if (i0 < L) *reinterpret_cast<uint32_t*>(a.dq + (size_t)(tok0 + i0) * a.ld + col) = pack_bf16(dq[n][0], dq[n][1]);
        if (i1 < L) *reinterpret_cast<uint32_t*>(a.dq + (size_t)(tok0 + i1) * a.ld + col) = pack_bf16(dq[n][2], dq[n][3]);
    }
}

// backward dK/dV: CTA owns 64 keys ; tile roles 0 = K, 1 = V, 2 = Q, 3 = dO, 4 = O (streamed)
template <int DH, bool JAGGED>
__global__ void __launch_bounds__(ATT_THREADS) sas_attn_bwd_dkdv_kernel(SasAttnArgs a) {
    pdl_wait();
    a.drop.resolve();
    extern __shared__ __align__(16) unsigned char att_smem_raw[];
    SasSmem<DH>& sm = *reinterpret_cast<SasSmem<DH>*>(att_smem_raw);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int kt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int k0 = kt * ATT_BLK;
    long long tok0;
    int L;
    seq_span<JAGGED>(a.offsets, a.T, a.L, b, tok0, L);
    if (JAGGED && k0 >= L) return;   // key tile past the end of a packed sequence
    const int nqt = (L + ATT_BLK - 1) / ATT_BLK;

    att_load_tile<DH>(sm.tile[0], a.k + (size_t)tok0 * a.ld + h * DH, a.ld, 0, k0, L, 0, tid);
    att_load_tile<DH>(sm.tile[1], a.v + (size_t)tok0 * a.ld + h * DH, a.ld, 0, k0, L, 0, tid);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    uint32_t kf[DH / 16][4], vf[DH / 16][4];
    att_load_afrag<DH>(kf, sm.tile[0], warp * 16, lane);
    att_load_afrag<DH>(vf, sm.tile[1], warp * 16, lane);
    const int j0 = k0 + warp * 16 + g, j1 = j0 + 8;
    const bool kok0 = j0 < L && a.pad[tok0 + j0] == 0, kok1 = j1 < L && a.pad[tok0 + j1] == 0;
    float dk[DH / 8][4], dv[DH / 8][4];
#pragma unroll
    for (int n = 0; n < DH / 8; ++n)
#pragma unroll
        for (int r = 0; r < 4; ++r) dk[n][r] = 0.f, dv[n][r] = 0.f;

    for (int qt = kt; qt < nqt; ++qt) {
        const int q0 = qt * ATT_BLK;
        __syncthreads();
        att_load_tile<DH>(sm.tile[2], a.q + (size_t)tok0 * a.ld + h * DH, a.ld, 0, q0, L, 0, tid);
        att_load_tile<DH>(sm.tile[3], a.d_out + (size_t)tok0 * a.ld + h * DH, a.ld, 0, q0, L, 0, tid);
        att_load_tile<DH>(sm.tile[4], a.out + (size_t)tok0 * a.ld + h * DH, a.ld, 0, q0, L, 0, tid);
        cp_async_commit();
        if (tid < ATT_BLK) {
            int i = q0 + tid;
            sm.lse_tile[tid] = (i < L) ? a.lse[sas_lse_at<JAGGED>(a, b, h, tok0, L, i)] : 0.f;
            sm.pad_tile[tid] = (i < L) ? a.pad[tok0 + i] : 1;  // QUERY padding here
        }
        cp_async_wait<0>();
        __syncthreads();
        sas_rowdot<DH>(sm.dsum_tile, sm.tile[3], sm.tile[4], tid);
        __syncthreads();

        float st[8][4], dat[8][4];
#pragma unroll
        for (int n = 0; n < 8; ++n)
#pragma unroll
            for (int r = 0; r < 4; ++r) st[n][r] = 0.f, dat[n][r] = 0.f;
        att_mma_nt<DH>(st, kf, sm.tile[2], lane);
        att_mma_nt<DH>(dat, vf, sm.tile[3], lane);
#pragma unroll
        for (int n = 0; n < 8; ++n)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int il = n * 8 + 2 * t + (r & 1), i = q0 + il;
                const int j = (r < 2) ? j0 : j1;
                const bool valid = (j <= i) && (i < L) && ((r < 2) ? kok0 : kok1) && sm.pad_tile[il] == 0;
                float pd = 0.f, dsv = 0.f;
                if (valid) {
                    float p = __expf(st[n][r] * a.scale - sm.lse_tile[il]);
                    const uint32_t drow = sas_drop_row<JAGGED>(a, b, h, tok0, L, i);
                    pd = a.drop.apply(p, drow, (uint32_t)j);
                    float dA = a.drop.apply(dat[n][r], drow, (uint32_t)j);
                    dsv = p * (dA - sm.dsum_tile[il]) * a.scale;
                }
                st[n][r] = pd;
                dat[n][r] = dsv;
            }
        uint32_t pf[4][4];
        att_pack_p(pf, st);
        att_mma_nn<DH>(dv, pf, sm.tile[3], lane);
        att_pack_p(pf, dat);
        att_mma_nn<DH>(dk, pf, sm.tile[2], lane);
    }
#pragma unroll
    for (int n = 0; n < DH / 8; ++n) {
        int col = h * DH + n * 8 + 2 * t;
        if (j0 < L) {
            *reinterpret_cast<uint32_t*>(a.dk + (size_t)(tok0 + j0) * a.ld + col) = pack_bf16(dk[n][0], dk[n][1]);
            *reinterpret_cast<uint32_t*>(a.dv + (size_t)(tok0 + j0) * a.ld + col) = pack_bf16(dv[n][0], dv[n][1]);
        }
        if (j1 < L) {
            *reinterpret_cast<uint32_t*>(a.dk + (size_t)(tok0 + j1) * a.ld + col) = pack_bf16(dk[n][2], dk[n][3]);
            *reinterpret_cast<uint32_t*>(a.dv + (size_t)(tok0 + j1) * a.ld + col) = pack_bf16(dv[n][2], dv[n][3]);
        }
    }
}

}  // namespace grb
