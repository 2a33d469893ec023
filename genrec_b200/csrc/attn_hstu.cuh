// genrec_b200 - HSTU pointwise (SiLU) attention, forward and backward (mma.sync m16n8k16 path).
//
//   S[b,h,i,j] = Q_i . K_j + Wpos[pb(i-j), h] + Wtime[tb(|ts_i - ts_j|), h]
//   valid      = (j <= i) and not pad[b,j]
//   A          = valid ? silu(S) : 0          O = A V
// (reference: genrec/models/hstu.py:244-267; SURVEY.md Appendix A).  No [L,L] fp tensor ever reaches HBM.
//
// All integer work is hoisted out of the per-head / per-layer kernels: `hstu_bias_index_kernel` runs ONCE per batch and
// writes one uint16 per (b, i, j):  pb(i-j) * 64 + tb(|ts_i - ts_j|)  (tb = integer-threshold form of the reference's
// fp32 log / 0.693 expression), or the sentinel npos*64 when the cell is masked (j > i, padded key).  Each attention CTA
// builds, for its head, the table  wcomb[pb*64 + tb] = Wpos[pb,h] + Wtime[tb,h]  in shared memory with
// wcomb[sentinel] = -30000: silu(-30000) and silu'(-30000) are exactly 0 in fp32, so masking costs no instruction.
// The per-element work is then: one 16-bit index load, one table load, one add, the SiLU.
// The 10 MB index matrix (cfg-2) stays L2-resident and is shared by every head of every layer, forward and backward.
//
// Layout: Q/K/V/dO/O are row-major [T = B*L, ld] bf16 with head h at columns h*DH .. h*DH+DH-1.
// One CTA = 4 warps = 64 query rows (fwd, dQ) or 64 key rows (dK/dV); the other operand streams through shared memory
// in double-buffered 64-row tiles (cp.async).  Warps whose rows lie beyond L and 8-wide blocks above the causal diagonal
// are skipped (warp-uniform branches).
#pragma once
#include "common.cuh"

namespace grb {

constexpr int ATT_BLK = 64;       // rows per CTA and per streamed tile
constexpr int ATT_THREADS = 128;  // 4 warps x 16 rows
constexpr int ATT_MAX_BUCKETS = 64;
// Diagonal tiles that lie wholly below L also take the guard-free straight-line path: their masked (above-diagonal) cells are
// computed and come out as exact zeros through the sentinel index, which costs up to half a tile of wasted work but lets
// the scheduler interleave all 32 score chains of a lane.  (-DGRB_ATT_DIAG_FULL=0 restores the per-warp triangular skipping.)
#ifndef GRB_ATT_DIAG_FULL
#define GRB_ATT_DIAG_FULL 1
#endif
constexpr bool ATT_DIAG_FULL = GRB_ATT_DIAG_FULL != 0;
constexpr int ATT_IX_LD = ATT_BLK + 8;  // padded row (uint16 elements) of the index tile in smem: 144 B, conflict-free
constexpr float ATT_MASK_BIAS = -30000.f;

struct HstuBiasArgs {
    const float* wpos;           // [npos, H]
    const float* wtime;          // [ntime, H] or null
    const uint16_t* bias_index;  // [B, L, ldix]
    int ldix;                    // elements, multiple of 8
    int npos, ntime;
    int pos_uniform;             // 1: every delta in [0, L) maps to pos bucket `pos_bucket0` (the reference's degenerate case)
    int pos_bucket0;
};

struct HstuAttnArgs {
    const bf16* q; const bf16* k; const bf16* v;   // forward operands (activations after SiLU)
    int ldq, ldk, ldv;
    int B, L, H;
    HstuBiasArgs bias;
    // forward
    bf16* o; int ldo;
    // backward
    const bf16* d_o; int lddo;
    const bf16* zq; const bf16* zk; const bf16* zv; int ldz;    // pre-activations (nullable -> no silu' factor)
    bf16* dq; bf16* dk; bf16* dv; int lddq;                       // gradients w.r.t. pre-activations (or activations if z null)
    float* dwpos;   // [npos, H]  accumulated (atomicAdd)
    float* dwtime;  // [ntime, H] accumulated
    float* dw_part; // nullable: [2H][B * key tiles][64] scratch for the ordered cross-CTA sum of dwpos / dwtime (det_finish_kernel)
};

GRB_DEVINL int time_bucket_dev(long long dt, const long long* thr, int ntime) {
    long long d = dt < 0 ? -dt : dt;
    d = d < 1 ? 1 : d;
    int e = 63 - __clzll(d);
    int b = e + (d >= thr[e + 1] ? 1 : 0);
    return min(b, ntime - 1);
}

// out[b, i, j] = (j <= i && !pad[b, j]) ? pos_bucket[i - j] * 64 + bucket(|ts[b,i] - ts[b,j]|) : npos * 64
// grid (ceil(ld / 256), ceil(L / 8), B), block 256 = 8 query rows x 32 threads ; a thread produces 8 neighbouring key
// columns and writes them with one 16-byte store (ld % 8 == 0).
__global__ void __launch_bounds__(256) hstu_bias_index_kernel(const long long* __restrict__ ts, const uint8_t* __restrict__ pad,
                                                             const long long* __restrict__ thr_g, const uint8_t* __restrict__ pos_bucket,
                                                             int L, int ld, int npos, int ntime, uint16_t* __restrict__ out) {
    pdl_wait();
    __shared__ long long thr[ATT_MAX_BUCKETS + 1];
    for (int i = threadIdx.x; i <= ATT_MAX_BUCKETS; i += 256) thr[i] = thr_g[i];
    __syncthreads();
    const int b = blockIdx.z, i = blockIdx.y * 8 + (threadIdx.x >> 5), j0 = (blockIdx.x * 32 + (threadIdx.x & 31)) * 8;
    if (i >= L || j0 >= ld) return;
    const size_t row = (size_t)b * L;
    const unsigned masked = (unsigned)npos * 64u;
    const bool timed = ts != nullptr && ntime > 0;
    const long long ti = timed ? ts[row + i] : 0;
    unsigned v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const int j = j0 + k;
        v[k] = masked;
        if (j <= i && pad[row + j] == 0) {     // j <= i < L
            const unsigned tb = timed ? (unsigned)time_bucket_dev(ti - ts[row + j], thr, ntime) : 0u;
            v[k] = (unsigned)pos_bucket[i - j] * 64u + tb;
        }
    }
    uint4 o;
    o.x = v[0] | (v[1] << 16); o.y = v[2] | (v[3] << 16); o.z = v[4] | (v[5] << 16); o.w = v[6] | (v[7] << 16);
    *reinterpret_cast<uint4*>(out + (row + i) * ld + j0) = o;
}

template <int DH, int NFIXED = 2>
struct AttSmem {
    static constexpr int LD = DH + 8;
    bf16 fixed[NFIXED][ATT_BLK * LD]; // the CTA's own rows: Q (forward, NFIXED = 1: 44 KB -> five CTAs per SM at dh = 32) or Q, dO
    bf16 stream[2][2][ATT_BLK * LD];  // [buffer][operand] streamed tiles
    uint16_t ix[2][ATT_BLK * ATT_IX_LD];  // [buffer] index tile: [query row][key col]
};
// dynamic tail after AttSmem: float wcomb[npos*64 + 1] ; (dK/dV only) lane-private histograms

// cooperative 64 x DH tile load (rows row0.. of one batch element, zero-filled beyond L).  The 64-bit part of the address
// (g + tok0 * ld + col0) is folded into `g` once per kernel by the caller; inside, offsets are 32-bit and the loop is
// fully unrolled (the generic version spent ~30 integer instructions per 16-byte copy).
template <int DH>
GRB_DEVINL void att_load_tile(bf16* s, const bf16* gb, int ld, long long /*tok0 folded into gb*/, int row0, int L, int /*col0 folded*/, int tid) {
    constexpr int LD = DH + 8;
    constexpr int CH = DH / 8;  // 16-byte chunks per row
    constexpr int PER = ATT_BLK * CH / ATT_THREADS;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
        const int c = tid + i * ATT_THREADS;
        const int r = c / CH, kc = (c % CH) * 8;
        const int row = row0 + r;
        const bool ok = row < L;
        cp_async16(s + r * LD + kc, gb + (ok ? row * ld + kc : 0), ok ? 16 : 0);
    }
}
// 64 x 64 uint16 tile of the index matrix: rows q0.., cols k0.. ; everything out of range reads as `sentinel`
// (gb = bias_index + tok0 * ldix, folded once per kernel)
GRB_DEVINL void att_load_ix(uint16_t* s, const uint16_t* gb, int ldix, long long, int q0, int k0, int L, unsigned sentinel, int tid) {
    const unsigned s2 = sentinel | (sentinel << 16);
#pragma unroll
    for (int i = 0; i < ATT_BLK * 8 / ATT_THREADS; ++i) {
        const int c = tid + i * ATT_THREADS;
        const int r = c >> 3, kc = (c & 7) * 8;
        const bool ok = (q0 + r) < L && (k0 + kc) < ldix;
        if (ok) cp_async16(s + r * ATT_IX_LD + kc, gb + (q0 + r) * ldix + k0 + kc, 16);
        else *reinterpret_cast<uint4*>(s + r * ATT_IX_LD + kc) = make_uint4(s2, s2, s2, s2);
    }
}
// wcomb[pb*64 + tb] = Wpos[pb,h] + Wtime[tb,h] ; wcomb[npos*64] = mask
GRB_DEVINL void att_build_table(float* wcomb, const HstuBiasArgs& b, int h, int H, int tid) {
    const int n = b.npos * 64;
    for (int i = tid; i < n; i += ATT_THREADS) {
        const int pb = i >> 6, tb = i & 63;
        float v = b.wpos[pb * H + h];
        if (b.wtime && tb < b.ntime) v += b.wtime[tb * H + h];
        wcomb[i] = v;
    }
    if (tid == 0) wcomb[n] = ATT_MASK_BIAS;
}

// A-operand fragments of a 16 x DH slab (rows wrow..wrow+15 of an smem tile)
template <int DH>
GRB_DEVINL void att_load_afrag(uint32_t (&f)[DH / 16][4], const bf16* tile, int wrow, int lane) {
    constexpr int LD = DH + 8;
#pragma unroll
    for (int ks = 0; ks < DH / 16; ++ks) ldsm_x4(f[ks], tile + (wrow + lane_a_row(lane)) * LD + ks * 16 + lane_a_col(lane));
}

// acc[8][4] (16 rows x 64 cols) = Afrag(16 x DH) * Tile^T   where Tile is [64][DH] (k = DH contiguous); only the first
// `npairs` pairs of 8-column blocks are computed (warp-uniform), the others are set to 0.  acc is OVERWRITTEN.
template <int DH>
GRB_DEVINL void att_mma_nt(float (&acc)[8][4], const uint32_t (&af)[DH / 16][4], const bf16* tile, int lane, int npairs = 4) {
    constexpr int LD = DH + 8;
#pragma unroll
    for (int ks = 0; ks < DH / 16; ++ks) {
#pragma unroll
        for (int j2 = 0; j2 < 4; ++j2) {
            if (j2 < npairs) {
                uint32_t r[4];
                ldsm_x4(r, tile + (j2 * 16 + lane_b_row(lane)) * LD + ks * 16 + lane_b_col(lane));
                if (ks == 0) {
                    mma_bf16_z(acc[2 * j2], af[ks], r[0], r[1]);
                    mma_bf16_z(acc[2 * j2 + 1], af[ks], r[2], r[3]);
                } else {
                    mma_bf16(acc[2 * j2], af[ks], r[0], r[1]);
                    mma_bf16(acc[2 * j2 + 1], af[ks], r[2], r[3]);
                }
            } else if (ks == 0) {
#pragma unroll
                for (int r = 0; r < 4; ++r) acc[2 * j2][r] = 0.f, acc[2 * j2 + 1][r] = 0.f;
            }
        }
    }
}

// out[DH/8][4] (16 rows x DH cols) += P(16 x 64, as 4 k16 A-fragments) * Tile   where Tile is [64][DH] (n = DH contiguous)
// only k16 blocks [kbeg, kend) contribute (warp-uniform)
template <int DH>
GRB_DEVINL void att_mma_nn(float (&out)[DH / 8][4], const uint32_t (&pf)[4][4], const bf16* tile, int lane, int kbeg = 0, int kend = 4) {
    constexpr int LD = DH + 8;
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        if (kk >= kbeg && kk < kend) {
#pragma unroll
            for (int n2 = 0; n2 < DH / 16; ++n2) {
                uint32_t r[4];
                ldsm_x4_t(r, tile + (kk * 16 + lane_a_row(lane)) * LD + n2 * 16 + lane_a_col(lane));
                mma_bf16(out[2 * n2], pf[kk], r[0], r[1]);
                mma_bf16(out[2 * n2 + 1], pf[kk], r[2], r[3]);
            }
        }
    }
}

template <bool B>
struct FullTile {
    static constexpr bool value = B;
};

GRB_DEVINL void att_pack_p(uint32_t (&pf)[4][4], const float (&s)[8][4]) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        pf[kk][0] = pack_bf16(s[2 * kk][0], s[2 * kk][1]);
        pf[kk][1] = pack_bf16(s[2 * kk][2], s[2 * kk][3]);
        pf[kk][2] = pack_bf16(s[2 * kk + 1][0], s[2 * kk + 1][1]);
        pf[kk][3] = pack_bf16(s[2 * kk + 1][2], s[2 * kk + 1][3]);
    }
}

// ============================================================================================ forward
// fixed[0] = Q ; stream[buf] = {K, V}
template <int DH>
__global__ void __launch_bounds__(ATT_THREADS, DH == 32 ? 5 : 3) hstu_attn_fwd_kernel(HstuAttnArgs a) {
    pdl_wait();
    extern __shared__ __align__(16) unsigned char att_smem_raw[];
    AttSmem<DH, 1>& sm = *reinterpret_cast<AttSmem<DH, 1>*>(att_smem_raw);
    float* wcomb = reinterpret_cast<float*>(att_smem_raw + sizeof(AttSmem<DH, 1>));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int L = a.L, q0 = qt * ATT_BLK;
    const long long tok0 = (long long)b * L;
    const unsigned sentinel = (unsigned)a.bias.npos * 64u;

    att_build_table(wcomb, a.bias, h, a.H, tid);
    const bf16* gq = a.q + (size_t)tok0 * a.ldq + h * DH;
    const bf16* gk = a.k + (size_t)tok0 * a.ldk + h * DH;
    const bf16* gv = a.v + (size_t)tok0 * a.ldv + h * DH;
    const uint16_t* gix = a.bias.bias_index + (size_t)tok0 * a.bias.ldix;
    att_load_tile<DH>(sm.fixed[0], gq, a.ldq, 0, q0, L, 0, tid);
    auto load_stream = [&](int kt, int buf) {
        att_load_tile<DH>(sm.stream[buf][0], gk, a.ldk, 0, kt * ATT_BLK, L, 0, tid);
        att_load_tile<DH>(sm.stream[buf][1], gv, a.ldv, 0, kt * ATT_BLK, L, 0, tid);
        att_load_ix(sm.ix[buf], gix, a.bias.ldix, 0, q0, kt * ATT_BLK, L, sentinel, tid);
    };
    load_stream(0, 0);
    cp_async_commit();

    const int i0 = q0 + warp * 16 + g, i1 = i0 + 8;
    const bool warp_live = q0 + warp * 16 < L;  // warp-uniform
    uint32_t qf[DH / 16][4];
    float o[DH / 8][4];
#pragma unroll
    for (int n = 0; n < DH / 8; ++n)
#pragma unroll
        for (int r = 0; r < 4; ++r) o[n][r] = 0.f;

    for (int kt = 0; kt <= qt; ++kt) {
        const int buf = kt & 1;
        if (kt < qt) {
            load_stream(kt + 1, buf ^ 1);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();  // tile kt (and, first time, Q + table) visible to everyone
        if (kt == 0) att_load_afrag<DH>(qf, sm.fixed[0], warp * 16, lane);
        if (warp_live) {
            int nblk = (kt == qt) ? min(8, 2 * warp + 2) : 8;  // 8-key blocks intersecting this warp's causal triangle
            nblk = min(nblk, (L - kt * ATT_BLK + 7) >> 3);       // ... and lying below L
            const int npairs_rt = (nblk + 1) >> 1;
            // FULL: the whole 64-key tile is visible to this warp (every tile but the diagonal and the last one) - no
            // per-block guards, so the 32 score chains of a lane are one straight-line block the scheduler can interleave
            auto tile = [&](auto full_c) {
                constexpr bool FULL = decltype(full_c)::value;
                const int npairs = FULL ? 4 : npairs_rt;
                float s[8][4];
                att_mma_nt<DH>(s, qf, sm.stream[buf][0], lane, npairs);
                const uint16_t* ix = sm.ix[buf];
#pragma unroll
                for (int n = 0; n < 8; ++n) {
                    if (FULL || n < 2 * npairs) {
#pragma unroll
                        for (int hf = 0; hf < 2; ++hf) {
                            const uint32_t i2 = *reinterpret_cast<const uint32_t*>(ix + (warp * 16 + g + 8 * hf) * ATT_IX_LD + n * 8 + 2 * t);
                            s[n][2 * hf] = siluf(s[n][2 * hf] + wcomb[i2 & 0xffffu]);
                            s[n][2 * hf + 1] = siluf(s[n][2 * hf + 1] + wcomb[i2 >> 16]);
                        }
                    }
                }
                uint32_t pf[4][4];
                att_pack_p(pf, s);
                att_mma_nn<DH>(o, pf, sm.stream[buf][1], lane, 0, npairs);
            };
            if (npairs_rt == 4 || (ATT_DIAG_FULL && (kt + 1) * ATT_BLK <= L)) tile(FullTile<true>{}); else tile(FullTile<false>{});
        }
        __syncthreads();  // everyone done with buffer `buf` before it is refilled two iterations later
    }

#pragma unroll
    for (int n = 0; n < DH / 8; ++n) {
        int col = h * DH + n * 8 + 2 * t;
        if (i0 < L) *reinterpret_cast<uint32_t*>(a.o + (size_t)(tok0 + i0) * a.ldo + col) = pack_bf16(o[n][0], o[n][1]);
        if (i1 < L) *reinterpret_cast<uint32_t*>(a.o + (size_t)(tok0 + i1) * a.ldo + col) = pack_bf16(o[n][2], o[n][3]);
    }
}

// ============================================================================================ backward: dQ
// fixed = {Q, dO} ; stream[buf] = {K, V}
template <int DH>
__global__ void __launch_bounds__(ATT_THREADS, DH == 32 ? 4 : 2) hstu_attn_bwd_dq_kernel(HstuAttnArgs a) {
    pdl_wait();
    extern __shared__ __align__(16) unsigned char att_smem_raw[];
    AttSmem<DH>& sm = *reinterpret_cast<AttSmem<DH>*>(att_smem_raw);
    float* wcomb = reinterpret_cast<float*>(att_smem_raw + sizeof(AttSmem<DH>));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int L = a.L, q0 = qt * ATT_BLK;
    const long long tok0 = (long long)b * L;
    const unsigned sentinel = (unsigned)a.bias.npos * 64u;

    att_build_table(wcomb, a.bias, h, a.H, tid);
    const bf16* gq = a.q + (size_t)tok0 * a.ldq + h * DH;
    const bf16* gdo = a.d_o + (size_t)tok0 * a.lddo + h * DH;
    const bf16* gk = a.k + (size_t)tok0 * a.ldk + h * DH;
    const bf16* gv = a.v + (size_t)tok0 * a.ldv + h * DH;
    const uint16_t* gix = a.bias.bias_index + (size_t)tok0 * a.bias.ldix;
    att_load_tile<DH>(sm.fixed[0], gq, a.ldq, 0, q0, L, 0, tid);
    att_load_tile<DH>(sm.fixed[1], gdo, a.lddo, 0, q0, L, 0, tid);
    auto load_stream = [&](int kt, int buf) {
        att_load_tile<DH>(sm.stream[buf][0], gk, a.ldk, 0, kt * ATT_BLK, L, 0, tid);
        att_load_tile<DH>(sm.stream[buf][1], gv, a.ldv, 0, kt * ATT_BLK, L, 0, tid);
        att_load_ix(sm.ix[buf], gix, a.bias.ldix, 0, q0, kt * ATT_BLK, L, sentinel, tid);
    };
    load_stream(0, 0);
    cp_async_commit();

    const int i0 = q0 + warp * 16 + g, i1 = i0 + 8;
    const bool warp_live = q0 + warp * 16 < L;
    {   // the epilogue multiplies by silu'(zq) of the warp's 16 query rows: pull those row segments towards L2 now
        const int ir = q0 + warp * 16 + (lane & 15);
        if (a.zq != nullptr && lane < 16 && ir < L) prefetch_l2(a.zq + (size_t)(tok0 + ir) * a.ldz + h * DH);
    }
    uint32_t qf[DH / 16][4], dof[DH / 16][4];
    float dq[DH / 8][4];
#pragma unroll
    for (int n = 0; n < DH / 8; ++n)
#pragma unroll
        for (int r = 0; r < 4; ++r) dq[n][r] = 0.f;

    for (int kt = 0; kt <= qt; ++kt) {
        const int buf = kt & 1;
        if (kt < qt) {
            load_stream(kt + 1, buf ^ 1);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (kt == 0) {
            att_load_afrag<DH>(qf, sm.fixed[0], warp * 16, lane);
            att_load_afrag<DH>(dof, sm.fixed[1], warp * 16, lane);
        }
        if (warp_live) {
            int nblk = (kt == qt) ? min(8, 2 * warp + 2) : 8;
            nblk = min(nblk, (L - kt * ATT_BLK + 7) >> 3);
            const int npairs_rt = (nblk + 1) >> 1;
            auto tile = [&](auto full_c) {     // FULL: no per-block guards (see the forward kernel)
                constexpr bool FULL = decltype(full_c)::value;
                const int npairs = FULL ? 4 : npairs_rt;
                float s[8][4], da[8][4];
                att_mma_nt<DH>(s, qf, sm.stream[buf][0], lane, npairs);    // S  = Q K^T
                att_mma_nt<DH>(da, dof, sm.stream[buf][1], lane, npairs);  // dA = dO V^T
                const uint16_t* ix = sm.ix[buf];
#pragma unroll
                for (int n = 0; n < 8; ++n) {
                    if (FULL || n < 2 * npairs) {
#pragma unroll
                        for (int hf = 0; hf < 2; ++hf) {
                            const uint32_t i2 = *reinterpret_cast<const uint32_t*>(ix + (warp * 16 + g + 8 * hf) * ATT_IX_LD + n * 8 + 2 * t);
                            s[n][2 * hf] = da[n][2 * hf] * dsiluf(s[n][2 * hf] + wcomb[i2 & 0xffffu]);              // dS
                            s[n][2 * hf + 1] = da[n][2 * hf + 1] * dsiluf(s[n][2 * hf + 1] + wcomb[i2 >> 16]);
                        }
                    }
                }
                uint32_t pf[4][4];
                att_pack_p(pf, s);
                att_mma_nn<DH>(dq, pf, sm.stream[buf][0], lane, 0, npairs);  // dQ += dS K
            };
            if (npairs_rt == 4 || (ATT_DIAG_FULL && (kt + 1) * ATT_BLK <= L)) tile(FullTile<true>{}); else tile(FullTile<false>{});
        }
        __syncthreads();
    }

#pragma unroll
    for (int n = 0; n < DH / 8; ++n) {
        int col = h * DH + n * 8 + 2 * t;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            int i = half ? i1 : i0;
            if (i >= L) continue;
            float v0 = dq[n][2 * half], v1 = dq[n][2 * half + 1];
            if (a.zq) {
                float2 z = unpack_bf16(*reinterpret_cast<const uint32_t*>(a.zq + (size_t)(tok0 + i) * a.ldz + col));
                v0 *= dsiluf(z.x);
                v1 *= dsiluf(z.y);
            }
            *reinterpret_cast<uint32_t*>(a.dq + (size_t)(tok0 + i) * a.lddq + col) = pack_bf16(v0, v1);
        }
    }
}

// ============================================================================================ backward: dK, dV, bias tables
// CTA owns 64 keys: fixed = {K, V} ; stream[buf] = {Q, dO}
// K and V are only needed as register fragments, so they are staged through stream buffer 1 before the main loop.
// dynamic smem tail: wcomb[npos*64+1] (padded to 16 B) then LANE-PRIVATE histograms hist_t[4][ntime+1][32], hist_p[4][npos+1][32]
// (each lane owns one 4-byte column: plain read-modify-write, bank-conflict free, no atomics; hist_p only when the
// position buckets are not uniform)
template <int DH>
struct AttSmemKV {
    static constexpr int LD = DH + 8;
    bf16 stream[2][2][ATT_BLK * LD];
    uint16_t ix[2][ATT_BLK * ATT_IX_LD];
};
// HAS_TIME / POS_UNI are compile-time so that the per-cell histogram code carries no branches
template <int DH, bool HAS_TIME, bool POS_UNI>
__global__ void __launch_bounds__(ATT_THREADS, DH == 32 ? 3 : 2) hstu_attn_bwd_dkdv_kernel(HstuAttnArgs a, int table_bytes) {
    pdl_wait();
    extern __shared__ __align__(16) unsigned char att_smem_raw[];
    AttSmemKV<DH>& sm = *reinterpret_cast<AttSmemKV<DH>*>(att_smem_raw);
    float* wcomb = reinterpret_cast<float*>(att_smem_raw + sizeof(AttSmemKV<DH>));
    float* hist_t = reinterpret_cast<float*>(att_smem_raw + sizeof(AttSmemKV<DH>) + table_bytes);
    const int ntime = a.bias.ntime, npos = a.bias.npos;
    const int nt_bins = ntime + 1;   // + one spare bin: masked cells of the uniform-position layout index it with an exact 0
    float* hist_p = hist_t + 4 * nt_bins * 32;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int kt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
    const int L = a.L, k0 = kt * ATT_BLK;
    const long long tok0 = (long long)b * L;
    constexpr bool has_time = HAS_TIME, pos_uniform = POS_UNI;
    const int nqt = (L + ATT_BLK - 1) / ATT_BLK;
    const unsigned sentinel = (unsigned)npos * 64u;

    att_build_table(wcomb, a.bias, h, a.H, tid);
    for (int i = tid; i < 4 * (nt_bins + (pos_uniform ? 0 : npos + 1)) * 32; i += ATT_THREADS) hist_t[i] = 0.f;
    const bf16* gq = a.q + (size_t)tok0 * a.ldq + h * DH;
    const bf16* gdo = a.d_o + (size_t)tok0 * a.lddo + h * DH;
    const bf16* gk = a.k + (size_t)tok0 * a.ldk + h * DH;
    const bf16* gv = a.v + (size_t)tok0 * a.ldv + h * DH;
    const uint16_t* gix = a.bias.bias_index + (size_t)tok0 * a.bias.ldix;
    att_load_tile<DH>(sm.stream[1][0], gk, a.ldk, 0, k0, L, 0, tid);
    att_load_tile<DH>(sm.stream[1][1], gv, a.ldv, 0, k0, L, 0, tid);
    auto load_stream = [&](int qt, int buf) {
        att_load_tile<DH>(sm.stream[buf][0], gq, a.ldq, 0, qt * ATT_BLK, L, 0, tid);
        att_load_tile<DH>(sm.stream[buf][1], gdo, a.lddo, 0, qt * ATT_BLK, L, 0, tid);
        att_load_ix(sm.ix[buf], gix, a.bias.ldix, 0, qt * ATT_BLK, k0, L, sentinel, tid);
    };
    load_stream(kt, 0);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();
    uint32_t kf[DH / 16][4], vf[DH / 16][4];
    att_load_afrag<DH>(kf, sm.stream[1][0], warp * 16, lane);
    att_load_afrag<DH>(vf, sm.stream[1][1], warp * 16, lane);
    __syncthreads();  // K/V fragments are in registers: stream buffer 1 may now be refilled
    const int j0 = k0 + warp * 16 + g, j1 = j0 + 8;
    const bool warp_live = k0 + warp * 16 < L;
    {   // the epilogue multiplies by silu'(z) of the warp's 16 key rows: pull those 64-byte row segments towards L2 now
        const int jr = k0 + warp * 16 + (lane & 15);
        const bf16* zsrc = (lane < 16) ? a.zk : a.zv;
        if (zsrc != nullptr && jr < L) prefetch_l2(zsrc + (size_t)(tok0 + jr) * a.ldz + h * DH);
    }
    float dk[DH / 8][4], dv[DH / 8][4];
#pragma unroll
    for (int n = 0; n < DH / 8; ++n)
#pragma unroll
        for (int r = 0; r < 4; ++r) dk[n][r] = 0.f, dv[n][r] = 0.f;
    float* my_ht = hist_t + (warp * nt_bins) * 32 + lane;
    float* my_hp = hist_p + (warp * (npos + 1)) * 32 + lane;   // bin `npos` only ever receives the zeros of masked cells
    float pos_acc = 0.f;  // sum of dS when all cells share one position bucket

    for (int qt = kt; qt < nqt; ++qt) {
        const int buf = (qt - kt) & 1;
        if (qt + 1 < nqt) {
            load_stream(qt + 1, buf ^ 1);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (warp_live) {
            // query 8-blocks that can see this warp's keys (diagonal tile: queries >= first key of the warp)
            const int nb0_rt = (qt == kt) ? 2 * warp : 0;  // first live 8-query block (warp-uniform, even)
            const int nb1_rt = min(8, (L - qt * ATT_BLK + 7) >> 3);   // query blocks at or beyond L hold nothing (last tile of a short sequence)
            auto tile = [&](auto full_c) {     // FULL: all 8 query blocks are live - no per-block guards (see the forward kernel)
                constexpr bool FULL = decltype(full_c)::value;
                const int nb0 = FULL ? 0 : nb0_rt, nb1 = FULL ? 8 : nb1_rt;
                const int kb0 = nb0 >> 1;                    // first live k16 block for the second GEMMs
                const int kb1 = (nb1 + 1) >> 1;
                float st[8][4], dat[8][4];
                att_mma_nt<DH>(st, kf, sm.stream[buf][0], lane, kb1);   // S^T  = K Q^T   (rows = keys, cols = queries)
                att_mma_nt<DH>(dat, vf, sm.stream[buf][1], lane, kb1);  // dA^T = V dO^T
                const uint16_t* ix = sm.ix[buf];
                // pass 1 - independent per cell (the compiler interleaves the chains): A^T and dS^T in place
#pragma unroll
                for (int n = 0; n < 8; ++n) {
                    if (FULL || (n >= nb0 && n < nb1)) {
#pragma unroll
                        for (int r = 0; r < 4; ++r) {
                            const int il = n * 8 + 2 * t + (r & 1);
                            const int jl = warp * 16 + g + ((r < 2) ? 0 : 8);
                            const unsigned id = ix[il * ATT_IX_LD + jl];
                            const float x = st[n][r] + wcomb[id];
                            const float sg = sigmoidf_fast(x);
                            const float dsv = dat[n][r] * (sg * (1.f + x * (1.f - sg)));   // exactly 0 on masked cells
                            st[n][r] = x * sg;
                            dat[n][r] = dsv;
                            pos_acc += dsv;
                        }
                    } else {
#pragma unroll
                        for (int r = 0; r < 4; ++r) st[n][r] = 0.f, dat[n][r] = 0.f;
                    }
                }
                // pass 2 - bias-table gradients: scatter dS into the lane-private histograms.  Kept apart from pass 1 because
                // the read-modify-writes may alias each other (two cells of a lane often share a bucket) and would otherwise
                // serialise the whole element-wise chain behind them.  Masked cells carry dS == 0 exactly and index a valid
                // (spare) bin, so no branch is needed.
                if (has_time || !pos_uniform) {
#pragma unroll
                    for (int n = 0; n < 8; ++n) {
                        if (FULL || (n >= nb0 && n < nb1)) {
#pragma unroll
                            for (int r = 0; r < 4; ++r) {
                                const int il = n * 8 + 2 * t + (r & 1);
                                const int jl = warp * 16 + g + ((r < 2) ? 0 : 8);
                                const unsigned id = ix[il * ATT_IX_LD + jl];
                                if (has_time) my_ht[(pos_uniform ? id : (id & 63u)) * 32] += dat[n][r];   // uniform layout: id = time bucket, 64 = masked
                                if (!pos_uniform) my_hp[(id >> 6) * 32] += dat[n][r];
                            }
                        }
                    }
                }
                uint32_t pf[4][4];
                att_pack_p(pf, st);
                att_mma_nn<DH>(dv, pf, sm.stream[buf][1], lane, kb0, kb1);  // dV += A^T dO
                att_pack_p(pf, dat);
                att_mma_nn<DH>(dk, pf, sm.stream[buf][0], lane, kb0, kb1);  // dK += dS^T Q
            };
            if ((nb0_rt == 0 || ATT_DIAG_FULL) && nb1_rt == 8) tile(FullTile<true>{}); else tile(FullTile<false>{});
        }
        __syncthreads();
    }

#pragma unroll
    for (int n = 0; n < DH / 8; ++n) {
        int col = h * DH + n * 8 + 2 * t;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            int j = half ? j1 : j0;
            if (j >= L) continue;
            float k0v = dk[n][2 * half], k1v = dk[n][2 * half + 1];
            float v0v = dv[n][2 * half], v1v = dv[n][2 * half + 1];
            size_t zo = (size_t)(tok0 + j) * a.ldz + col;
            if (a.zk) {
                float2 z = unpack_bf16(*reinterpret_cast<const uint32_t*>(a.zk + zo));
                k0v *= dsiluf(z.x);
                k1v *= dsiluf(z.y);
            }
            if (a.zv) {
                float2 z = unpack_bf16(*reinterpret_cast<const uint32_t*>(a.zv + zo));
                v0v *= dsiluf(z.x);
                v1v *= dsiluf(z.y);
            }
            size_t go = (size_t)(tok0 + j) * a.lddq + col;
            *reinterpret_cast<uint32_t*>(a.dk + go) = pack_bf16(k0v, k1v);
            *reinterpret_cast<uint32_t*>(a.dv + go) = pack_bf16(v0v, v1v);
        }
    }

    // bias-table gradients: per-CTA sums, added across the CTAs of a head in (sequence, key tile) order when dw_part is given
    __shared__ float s_pos[ATT_THREADS / 32];
    if (pos_uniform) {
        pos_acc = warp_sum(pos_acc);
        if (lane == 0) s_pos[warp] = pos_acc;
    }
    __syncthreads();
    const int member = b * gridDim.x + kt, nmem = gridDim.x * gridDim.z;
    auto pos_sum = [&](int) {
        float v = 0.f;
        for (int w = 0; w < ATT_THREADS / 32; ++w) v += s_pos[w];
        return v;
    };
    auto pos_bin = [&](int bk) {
        float v = 0.f;
        for (int w = 0; w < 4; ++w)
            for (int l = 0; l < 32; ++l) v += hist_p[(w * (npos + 1) + bk) * 32 + l];
        return v;
    };
    auto time_bin = [&](int bk) {
        float v = 0.f;
        for (int w = 0; w < 4; ++w)
            for (int l = 0; l < 32; ++l) v += hist_t[(w * nt_bins + bk) * 32 + l];
        return v;
    };
    if (a.dw_part) {
        if (pos_uniform) det_store(a.dw_part, h, member, nmem, 64, 1, pos_sum);
        else det_store(a.dw_part, h, member, nmem, 64, npos, pos_bin);
        if (has_time && a.dwtime) det_store(a.dw_part, a.H + h, member, nmem, 64, ntime, time_bin);
    } else {
        if (pos_uniform) {
            if (tid == 0) atomicAdd(a.dwpos + a.bias.pos_bucket0 * a.H + h, pos_sum(0));
        } else {
            for (int bk = tid; bk < npos; bk += ATT_THREADS) atomicAdd(a.dwpos + bk * a.H + h, pos_bin(bk));
        }
        if (has_time && a.dwtime)
            for (int bk = tid; bk < ntime; bk += ATT_THREADS) atomicAdd(a.dwtime + bk * a.H + h, time_bin(bk));
    }
}

}  // namespace grb
