// genrec_b200 - T5-style attention core for TIGER (genrec/modules/transformer.py:44-159), forward and backward.
//
//   scores = (q k^T) * scale + rel_bias[h, bucket(j - i)]              (self-attention only)          transformer.py:136-141
//   scores = masked_fill(key_padding_mask, -1e9) ; scores += causal mask (-inf above the diagonal)     transformer.py:143-151
//   out    = dropout(softmax(scores)) v                                                               transformer.py:153-156
//
// TIGER's sequences are short (encoder 1 + 20 items x 3 tokens, decoder <= 4, head_dim 64) and the op is a few GFLOP per step, so
// this is an FP32 CUDA-core kernel with bf16 inputs / outputs (the tensors the wgmma projection GEMMs produce and consume):
// a CTA owns 32 query rows of one (batch, head); thread (row r, key quarter kq) walks the keys kq, kq + 4, ... of every 64-key
// tile with its own online-softmax state; the four states of a row are merged with shuffles.  Rectangular (cross-attention) and
// non-causal (encoder) shapes are the general case; the relative-position bucket of every delta = j - i is a host-made table.
// Backward: one pass per query tile recomputes the probabilities from the saved log-sum-exp; dQ stays in registers, the dK / dV
// contributions of the tile are reduced over its 32 query rows in shared memory.  With one or two query tiles they leave as one
// fp32 atomic per (key, d) onto zero, which commutes exactly; with more, each tile stores its partials and t5_dkdv_sum_kernel adds
// them in tile order.  The bias-table gradient is accumulated per CTA in shared-memory bins in a fixed order (each diagonal
// delta = j - i of a key tile in row order, then the diagonals of a bucket in delta order) and the CTAs' bins are added by
// det_finish, so two calls give the same bits.
//
// Packed (jagged) batches: sequence b is rows offsets[b] .. offsets[b+1]-1 of T, clamped to [0, T) and to Lk = max_len (seq_span).
//   T5_PACKED_SELF  (encoder self-attention): queries and keys are the rows of one sequence; i and j count from its first row, so the
//                   bucket of j - i is the padded one when the pads follow the items.  Query tiles past a sequence's end exit at once
//                   (forward) or only store their zero bias bins / dK | dV partials (backward).  lse is per token, [H, T, 2], and the
//                   dropout row key is the query's token row: (row * H + h), column j.
//   T5_PACKED_CROSS (decoder cross-attention): queries stay dense [B, Lq]; the keys of b are its packed rows.  lse and the dropout
//                   keys are the padded ones, so the masks equal those of the padded batch whose pads follow the keys.
// No key padding in either.  The kernels write only sequence rows: the caller zeroes the idle rows of out (self), dq (self) and dk / dv.
// PACK is a template parameter, so the padded instantiations compile to the code they had before packed batches existed (up to
// the order of two independent register initialisations in the forward).  Loop bounds are written out inline below: behind a
// helper call the compiler rotates the padded key loops differently.
#pragma once
#include "common.cuh"
#include "tc_gemm.cuh"   // exp_accurate

namespace grb {

struct T5AttnArgs {
    const bf16* q; int ldq;          // [B, Lq, ldq], head h = columns h*DH ..
    const bf16* k; const bf16* v; int ldk, ldv;   // [B, Lk, ld]
    int B, Lq, Lk, H;
    const float* bias;               // [H, nb] or null (cross-attention)
    const int* bucket;               // [Lq + Lk - 1]: bucket of delta = j - i at index delta + Lq - 1 (null iff bias null)
    int nb;
    const unsigned char* key_pad;    // [B, Lk] 1 = padded key, or null
    int causal;                      // 1: keys j > i are excluded (the additive -inf mask of the decoder)
    float scale;
    Dropout drop;
    // forward
    bf16* out; int ldo;              // [B, Lq, ldo]
    float* lse;                      // [B, H, Lq, 2] {row max, sum of exp(s - max)}: kept apart - with a padded row the max is -1e9
                                     // and log(sum) would vanish in its rounding
    // backward
    const bf16* dout; int lddo;      // [B, Lq, lddo]
    bf16* dq; int lddq;              // [B, Lq, lddq]
    float* dk; float* dv;            // [B, Lk, H * DH] fp32, accumulated (zero before the launch)
    float* dbias;                    // [H, nb] accumulated, or null
};
// packed batches: offsets [B+1] on the device and T packed rows, with T5AttnArgs::Lk = max_len (and Lq = max_len for self-attention).
// A trailing kernel parameter, so that the padded kernels keep their parameter layout.
struct T5Packed {
    const long long* offsets;
    int T;
};

enum { T5_PADDED = 0, T5_PACKED_SELF = 1, T5_PACKED_CROSS = 2 };

// The rows of batch entry b.  Packed: queries q0 .. q0 + nq - 1 of q / out / dout / dq (self) and keys k0 .. k0 + nk - 1 of
// k / v / dk / dv.  The helpers below give the padded instantiations the very expressions they had before packed layouts existed.
struct T5Span {
    size_t q0, k0;
    int nq, nk;
};
template <int PACK>
GRB_DEVINL T5Span t5_span(const T5AttnArgs& a, const T5Packed& pk, int b) {
    T5Span sp{0, 0, 0, 0};
    if constexpr (PACK != T5_PADDED) {
        long long tok0;
        seq_span<true>(pk.offsets, pk.T, a.Lk, b, tok0, sp.nk);
        sp.k0 = (size_t)tok0;
        sp.q0 = PACK == T5_PACKED_SELF ? sp.k0 : (size_t)b * a.Lq;
        sp.nq = PACK == T5_PACKED_SELF ? sp.nk : a.Lq;
    }
    return sp;
}
template <int PACK> GRB_DEVINL size_t t5_qrow(const T5AttnArgs& a, const T5Span& sp, int b, int i) {
    if constexpr (PACK != T5_PADDED) return sp.q0 + i; else return (size_t)b * a.Lq + i;
}
template <int PACK> GRB_DEVINL size_t t5_krow(const T5AttnArgs& a, const T5Span& sp, int b, int j0, int jj) {
    if constexpr (PACK != T5_PADDED) return sp.k0 + j0 + jj; else return (size_t)b * a.Lk + j0 + jj;
}
// lse slot and dropout row key of query i
template <int PACK>
GRB_DEVINL size_t t5_lse_at(const T5AttnArgs& a, const T5Packed& pk, const T5Span& sp, int b, int h, int i) {
    if constexpr (PACK == T5_PACKED_SELF) return (size_t)h * pk.T + sp.q0 + i; else return ((size_t)b * a.H + h) * a.Lq + i;
}
template <int PACK>
GRB_DEVINL uint32_t t5_drop_row(const T5AttnArgs& a, const T5Span& sp, int b, int h, int i) {
    if constexpr (PACK == T5_PACKED_SELF) return ((uint32_t)sp.q0 + (uint32_t)i) * (uint32_t)a.H + (uint32_t)h;
    else return (uint32_t)(((size_t)b * a.H + h) * a.Lq + i);
}

constexpr int T5_ROWS = 32, T5_KEYS = 64, T5_THREADS = 128;

template <int DH, int PACK>
GRB_DEVINL void t5_load_tile(float* Ks, float* Vs, const T5AttnArgs& a, const T5Span& sp, int b, int h, int j0, int tid) {
    for (int e = tid; e < T5_KEYS * (DH / 8); e += T5_THREADS) {
        const int jj = e / (DH / 8), c = e % (DH / 8);
        float kf[8], vf[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) kf[i] = vf[i] = 0.f;
        if (j0 + jj < (PACK != T5_PADDED ? sp.nk : a.Lk)) {
            const uint4 ku = *reinterpret_cast<const uint4*>(a.k + t5_krow<PACK>(a, sp, b, j0, jj) * a.ldk + h * DH + c * 8);
            const uint4 vu = *reinterpret_cast<const uint4*>(a.v + t5_krow<PACK>(a, sp, b, j0, jj) * a.ldv + h * DH + c * 8);
            const float2 k0 = unpack_bf16(ku.x), k1 = unpack_bf16(ku.y), k2 = unpack_bf16(ku.z), k3 = unpack_bf16(ku.w);
            const float2 v0 = unpack_bf16(vu.x), v1 = unpack_bf16(vu.y), v2 = unpack_bf16(vu.z), v3 = unpack_bf16(vu.w);
            kf[0] = k0.x; kf[1] = k0.y; kf[2] = k1.x; kf[3] = k1.y; kf[4] = k2.x; kf[5] = k2.y; kf[6] = k3.x; kf[7] = k3.y;
            vf[0] = v0.x; vf[1] = v0.y; vf[2] = v1.x; vf[3] = v1.y; vf[4] = v2.x; vf[5] = v2.y; vf[6] = v3.x; vf[7] = v3.y;
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) { Ks[jj * (DH + 1) + c * 8 + i] = kf[i]; Vs[jj * (DH + 1) + c * 8 + i] = vf[i]; }
    }
}
template <int DH>
GRB_DEVINL void t5_load_row(float (&x)[DH], const bf16* p) {
#pragma unroll
    for (int c = 0; c < DH / 8; ++c) {
        const uint4 u = *reinterpret_cast<const uint4*>(p + c * 8);
        const float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y), f2 = unpack_bf16(u.z), f3 = unpack_bf16(u.w);
        x[c * 8] = f0.x; x[c * 8 + 1] = f0.y; x[c * 8 + 2] = f1.x; x[c * 8 + 3] = f1.y;
        x[c * 8 + 4] = f2.x; x[c * 8 + 5] = f2.y; x[c * 8 + 6] = f3.x; x[c * 8 + 7] = f3.y;
    }
}
// score of (i, j) as the reference builds it; returns false when the cell is excluded (causal)
GRB_DEVINL bool t5_score(const T5AttnArgs& a, const float* sbias, int b, int i, int j, float qk, float& s, bool& differentiable) {
    if (a.causal && j > i) return false;
    s = qk * a.scale;
    if (sbias) s += sbias[a.bucket[j - i + a.Lq - 1]];
    differentiable = true;
    if (a.key_pad && a.key_pad[(size_t)b * a.Lk + j]) { s = -1e9f; differentiable = false; }   // masked_fill: a constant
    return true;
}

// SPLIT_BH: (b, h) = blockIdx.z * gridDim.y + blockIdx.y, for B * H past the 65,535 CTAs gridDim.y allows; otherwise blockIdx.y
template <int DH, bool SPLIT_BH, int PACK = T5_PADDED>
__global__ void __launch_bounds__(T5_THREADS) t5_attn_fwd_kernel(T5AttnArgs a, T5Packed pk) {
    pdl_wait();
    a.drop.resolve();
    extern __shared__ float t5_smem[];
    float* Ks = t5_smem;                          // [64][DH + 1]
    float* Vs = Ks + T5_KEYS * (DH + 1);
    float* sbias = a.bias ? Vs + T5_KEYS * (DH + 1) : nullptr;   // [nb] this head's row of the table
    const int tid = threadIdx.x, r = tid >> 2, kq = tid & 3;
    const int bh = SPLIT_BH ? (int)(blockIdx.z * gridDim.y + blockIdx.y) : (int)blockIdx.y;
    if (SPLIT_BH && bh >= a.B * a.H) return;
    const int b = bh / a.H, h = bh % a.H;
    const T5Span sp = t5_span<PACK>(a, pk, b);
    if constexpr (PACK == T5_PACKED_SELF)
        if ((int)blockIdx.x * T5_ROWS >= sp.nq) return;   // query tile past the end of its sequence
    const int i = blockIdx.x * T5_ROWS + r;
    if (sbias) for (int e = tid; e < a.nb; e += T5_THREADS) sbias[e] = a.bias[h * a.nb + e];
    float q[DH], o[DH];
#pragma unroll
    for (int d = 0; d < DH; ++d) { q[d] = 0.f; o[d] = 0.f; }
    if (i < (PACK != T5_PADDED ? sp.nq : a.Lq)) t5_load_row<DH>(q, a.q + t5_qrow<PACK>(a, sp, b, i) * a.ldq + h * DH);
    float m = -INFINITY, l = 0.f;
    const uint32_t drow = t5_drop_row<PACK>(a, sp, b, h, i);
    for (int j0 = 0; j0 < (PACK != T5_PADDED ? sp.nk : a.Lk); j0 += T5_KEYS) {
        __syncthreads();
        t5_load_tile<DH, PACK>(Ks, Vs, a, sp, b, h, j0, tid);
        __syncthreads();
        if (i >= (PACK != T5_PADDED ? sp.nq : a.Lq)) continue;
        for (int jj = kq; jj < T5_KEYS && j0 + jj < (PACK != T5_PADDED ? sp.nk : a.Lk); jj += 4) {
            const float* kr = Ks + jj * (DH + 1);
            float qk = 0.f;
#pragma unroll
            for (int d = 0; d < DH; ++d) qk = fmaf(q[d], kr[d], qk);
            float s; bool diff;
            if (!t5_score(a, sbias, b, i, j0 + jj, qk, s, diff)) continue;
            if (s > m) {
                const float c = exp_accurate(m - s);   // m = -inf -> 0
                l *= c;
#pragma unroll
                for (int d = 0; d < DH; ++d) o[d] *= c;
                m = s;
            }
            const float p = exp_accurate(s - m);
            l += p;
            const float pd = a.drop.apply(p, drow, (uint32_t)(j0 + jj));
            const float* vr = Vs + jj * (DH + 1);
#pragma unroll
            for (int d = 0; d < DH; ++d) o[d] = fmaf(pd, vr[d], o[d]);
        }
    }
    // merge the four online-softmax states of the row
#pragma unroll
    for (int sh = 1; sh <= 2; sh <<= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m, sh), l2 = __shfl_xor_sync(0xffffffffu, l, sh);
        const float M = fmaxf(m, m2);
        const float c1 = M == -INFINITY ? 0.f : exp_accurate(m - M), c2 = M == -INFINITY ? 0.f : exp_accurate(m2 - M);
        l = l * c1 + l2 * c2;
#pragma unroll
        for (int d = 0; d < DH; ++d) o[d] = o[d] * c1 + __shfl_xor_sync(0xffffffffu, o[d], sh) * c2;
        m = M;
    }
    if (i < (PACK != T5_PADDED ? sp.nq : a.Lq)) {
        const float inv = l > 0.f ? __fdiv_rn(1.f, l) : 0.f;
        bf16* dst = a.out + t5_qrow<PACK>(a, sp, b, i) * a.ldo + h * DH;
#pragma unroll
        for (int d = 0; d < DH; d += 2)
            if (((d >> 1) & 3) == kq) *reinterpret_cast<uint32_t*>(dst + d) = pack_bf16(o[d] * inv, o[d + 1] * inv);
        if (kq == 0) reinterpret_cast<float2*>(a.lse)[t5_lse_at<PACK>(a, pk, sp, b, h, i)] = make_float2(m, l);
    }
}

constexpr int T5_DIAGS = T5_ROWS + T5_KEYS - 1;   // diagonals delta = j - i of a 32 x 64 tile

// dkv_part: [2][gridDim.x][K * H * DH] per-query-tile dK / dV partials when the grid has more than two query tiles, else null
// (atomics); K = B * Lk key rows, or T when packed.  db_part: [H][B * gridDim.x][nb] the bias bins of each CTA, non-null iff a.dbias is.
template <int DH, int PACK = T5_PADDED>
__global__ void __launch_bounds__(T5_THREADS) t5_attn_bwd_kernel(T5AttnArgs a, float* dkv_part, float* db_part, T5Packed pk) {
    pdl_wait();
    a.drop.resolve();
    extern __shared__ float t5_smem[];
    float* Ks = t5_smem;                                  // [64][DH + 1]
    float* Vs = Ks + T5_KEYS * (DH + 1);
    float* Qs = Vs + T5_KEYS * (DH + 1);                  // [32][DH + 1]
    float* dOs = Qs + T5_ROWS * (DH + 1);                 // [32][DH + 1]
    float* dSs = dOs + T5_ROWS * (DH + 1);                // [32][64 + 1]  dS (0 where not differentiable)
    float* Pds = dSs + T5_ROWS * (T5_KEYS + 1);           // [32][64 + 1]  dropped probabilities
    float* sdiag = Pds + T5_ROWS * (T5_KEYS + 1);         // [95] the tile's diagonal sums of dS
    int* sbk = reinterpret_cast<int*>(sdiag + T5_DIAGS);  // [95] their buckets (-1: outside the bucket map)
    float* sbias = sdiag + 2 * T5_DIAGS;                  // [nb]
    float* sdb = sbias + a.nb;                            // [nb] gradient bins of this CTA
    const int tid = threadIdx.x, r = tid >> 2, kq = tid & 3;
    const int b = blockIdx.y / a.H, h = blockIdx.y % a.H;
    const int i0 = blockIdx.x * T5_ROWS, i = i0 + r;
    const int D = a.H * DH;
    T5Span sp = t5_span<PACK>(a, pk, b);
    // a query tile past the end of its sequence adds nothing: it skips the keys, unless its zero partials must be stored
    if constexpr (PACK == T5_PACKED_SELF)
        if (i0 >= sp.nq && !dkv_part) sp.nk = 0;
    if (a.bias) for (int e = tid; e < a.nb; e += T5_THREADS) { sbias[e] = a.bias[h * a.nb + e]; sdb[e] = 0.f; }
    float q[DH], dO[DH], dq[DH];
#pragma unroll
    for (int d = 0; d < DH; ++d) { q[d] = 0.f; dO[d] = 0.f; dq[d] = 0.f; }
    float rmax = 0.f, rinv = 0.f, Dsum = 0.f;
    if (i < (PACK != T5_PADDED ? sp.nq : a.Lq)) {
        t5_load_row<DH>(q, a.q + t5_qrow<PACK>(a, sp, b, i) * a.ldq + h * DH);
        t5_load_row<DH>(dO, a.dout + t5_qrow<PACK>(a, sp, b, i) * a.lddo + h * DH);
        float o[DH];
        t5_load_row<DH>(o, a.out + t5_qrow<PACK>(a, sp, b, i) * a.ldo + h * DH);
#pragma unroll
        for (int d = 0; d < DH; ++d) Dsum = fmaf(dO[d], o[d], Dsum);   // rowsum(dO * O) = sum_j P_ij dP_ij
        const float2 ml = reinterpret_cast<const float2*>(a.lse)[t5_lse_at<PACK>(a, pk, sp, b, h, i)];
        rmax = ml.x; rinv = ml.y > 0.f ? __fdiv_rn(1.f, ml.y) : 0.f;
    }
    if (kq == 0) {
#pragma unroll
        for (int d = 0; d < DH; ++d) { Qs[r * (DH + 1) + d] = q[d]; dOs[r * (DH + 1) + d] = dO[d]; }
    }
    const uint32_t drow = t5_drop_row<PACK>(a, sp, b, h, i);
    for (int j0 = 0; j0 < (PACK != T5_PADDED ? sp.nk : a.Lk); j0 += T5_KEYS) {
        __syncthreads();
        t5_load_tile<DH, PACK>(Ks, Vs, a, sp, b, h, j0, tid);
        for (int e = tid; e < T5_ROWS * (T5_KEYS + 1); e += T5_THREADS) { dSs[e] = 0.f; Pds[e] = 0.f; }
        __syncthreads();
        if (i < (PACK != T5_PADDED ? sp.nq : a.Lq)) {
            for (int jj = kq; jj < T5_KEYS && j0 + jj < (PACK != T5_PADDED ? sp.nk : a.Lk); jj += 4) {
                const float* kr = Ks + jj * (DH + 1);
                const float* vr = Vs + jj * (DH + 1);
                float qk = 0.f, dov = 0.f;
#pragma unroll
                for (int d = 0; d < DH; ++d) { qk = fmaf(q[d], kr[d], qk); dov = fmaf(dO[d], vr[d], dov); }
                float s; bool diff;
                if (!t5_score(a, a.bias ? sbias : nullptr, b, i, j0 + jj, qk, s, diff)) continue;
                const float p = exp_accurate(s - rmax) * rinv;
                const float pd = a.drop.apply(p, drow, (uint32_t)(j0 + jj));           // = mask * keep_scale * p
                const float dp = p > 0.f ? dov * __fdiv_rn(pd, p) : 0.f;               // d loss / d P_ij
                const float ds = p * (dp - Dsum);
                Pds[r * (T5_KEYS + 1) + jj] = pd;
                if (diff) {
                    dSs[r * (T5_KEYS + 1) + jj] = ds;
                    const float dss = ds * a.scale;
#pragma unroll
                    for (int d = 0; d < DH; ++d) dq[d] = fmaf(dss, kr[d], dq[d]);
                }
            }
        }
        __syncthreads();
        // bias bins: thread t sums diagonal t (jj - r = t - 31) over the tile's rows in order, then each bin adds its diagonals in order
        if (a.dbias) {
            if (tid < T5_DIAGS) {
                float s = 0.f;
                for (int rr = 0; rr < T5_ROWS; ++rr) {
                    const int jj = tid - (T5_ROWS - 1) + rr;
                    if (jj >= 0 && jj < T5_KEYS) s += dSs[rr * (T5_KEYS + 1) + jj];
                }
                sdiag[tid] = s;
                const int idx = j0 + tid - (T5_ROWS - 1) - i0 + a.Lq - 1;   // delta + Lq - 1
                sbk[tid] = idx >= 0 && idx < a.Lq + a.Lk - 1 ? a.bucket[idx] : -1;
            }
            __syncthreads();
            for (int e = tid; e < a.nb; e += T5_THREADS) {
                float acc = sdb[e];
                for (int t = 0; t < T5_DIAGS; ++t)
                    if (sbk[t] == e) acc += sdiag[t];
                sdb[e] = acc;
            }
        }
        // dK_j += sum_r dS_rj scale q_r ; dV_j += sum_r Pd_rj dO_r : thread (key jj, half of the head dims)
        {
            const int jj = tid >> 1, half = tid & 1;
            if (j0 + jj < (PACK != T5_PADDED ? sp.nk : a.Lk)) {
                float gk[DH / 2], gv[DH / 2];
#pragma unroll
                for (int d = 0; d < DH / 2; ++d) { gk[d] = 0.f; gv[d] = 0.f; }
                for (int rr = 0; rr < T5_ROWS; ++rr) {
                    const float ds = dSs[rr * (T5_KEYS + 1) + jj] * a.scale, pd = Pds[rr * (T5_KEYS + 1) + jj];
                    const float* qr = Qs + rr * (DH + 1) + half * (DH / 2);
                    const float* gr = dOs + rr * (DH + 1) + half * (DH / 2);
#pragma unroll
                    for (int d = 0; d < DH / 2; ++d) { gk[d] = fmaf(ds, qr[d], gk[d]); gv[d] = fmaf(pd, gr[d], gv[d]); }
                }
                const size_t at = t5_krow<PACK>(a, sp, b, j0, jj) * D + h * DH + half * (DH / 2);
                if (dkv_part) {                           // this query tile's slot of the partials
                    size_t n;
                    if constexpr (PACK != T5_PADDED) n = (size_t)pk.T * D; else n = (size_t)a.B * a.Lk * D;
                    float4* dkp = reinterpret_cast<float4*>(dkv_part + blockIdx.x * n + at);
                    float4* dvp = reinterpret_cast<float4*>(dkv_part + (gridDim.x + blockIdx.x) * n + at);
#pragma unroll
                    for (int d = 0; d < DH / 8; ++d) {
                        dkp[d] = make_float4(gk[4 * d], gk[4 * d + 1], gk[4 * d + 2], gk[4 * d + 3]);
                        dvp[d] = make_float4(gv[4 * d], gv[4 * d + 1], gv[4 * d + 2], gv[4 * d + 3]);
                    }
                } else {                                  // at most two adds onto zero per element: exact in either order
#pragma unroll
                    for (int d = 0; d < DH / 2; ++d) { atomicAdd(a.dk + at + d, gk[d]); atomicAdd(a.dv + at + d, gv[d]); }
                }
            }
        }
    }
#pragma unroll
    for (int d = 0; d < DH; ++d) {
        dq[d] += __shfl_xor_sync(0xffffffffu, dq[d], 1);
        dq[d] += __shfl_xor_sync(0xffffffffu, dq[d], 2);
    }
    if (i < (PACK != T5_PADDED ? sp.nq : a.Lq)) {
        bf16* dst = a.dq + t5_qrow<PACK>(a, sp, b, i) * a.lddq + h * DH;
#pragma unroll
        for (int d = 0; d < DH; d += 2)
            if (((d >> 1) & 3) == kq) *reinterpret_cast<uint32_t*>(dst + d) = pack_bf16(dq[d], dq[d + 1]);
    }
    if (a.dbias) {
        __syncthreads();
        det_store(db_part, h, b * gridDim.x + blockIdx.x, a.B * gridDim.x, a.nb, a.nb, [&](int e) { return sdb[e]; });
    }
}

// dk / dv [n] = the dkv_part partials of t5_attn_bwd_kernel summed over its ntiles query tiles in tile order (n % 4 == 0)
__global__ void __launch_bounds__(256) t5_dkdv_sum_kernel(const float* part, int ntiles, size_t n, float* dk, float* dv) {
    pdl_wait();
    const size_t n4 = n / 4;
    for (size_t e = (size_t)blockIdx.x * 256 + threadIdx.x; e < 2 * n4; e += (size_t)gridDim.x * 256) {
        const int w = e >= n4;
        const size_t c = e - w * n4;
        const float4* p = reinterpret_cast<const float4*>(part + (size_t)w * ntiles * n) + c;
        float4 s = p[0];
        for (int t = 1; t < ntiles; ++t) {
            const float4 x = p[(size_t)t * n4];
            s.x += x.x; s.y += x.y; s.z += x.z; s.w += x.w;
        }
        reinterpret_cast<float4*>(w ? dv : dk)[c] = s;
    }
}

template <int DH>
inline size_t t5_fwd_smem(int nb) { return (size_t)(2 * T5_KEYS * (DH + 1) + nb) * sizeof(float); }
template <int DH>
inline size_t t5_bwd_smem(int nb) {
    return (size_t)(2 * T5_KEYS * (DH + 1) + 2 * T5_ROWS * (DH + 1) + 2 * T5_ROWS * (T5_KEYS + 1) + 2 * T5_DIAGS + 2 * nb) * sizeof(float);
}

}  // namespace grb
