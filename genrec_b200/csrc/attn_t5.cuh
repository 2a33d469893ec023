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
// contributions of the tile are reduced over its 32 query rows in shared memory and leave as one fp32 atomic per (key, d); the
// bias-table gradient is accumulated per CTA in shared memory bins.
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

constexpr int T5_ROWS = 32, T5_KEYS = 64, T5_THREADS = 128;

template <int DH>
GRB_DEVINL void t5_load_tile(float* Ks, float* Vs, const T5AttnArgs& a, int b, int h, int j0, int tid) {
    for (int e = tid; e < T5_KEYS * (DH / 8); e += T5_THREADS) {
        const int jj = e / (DH / 8), c = e % (DH / 8);
        float kf[8], vf[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) kf[i] = vf[i] = 0.f;
        if (j0 + jj < a.Lk) {
            const uint4 ku = *reinterpret_cast<const uint4*>(a.k + ((size_t)b * a.Lk + j0 + jj) * a.ldk + h * DH + c * 8);
            const uint4 vu = *reinterpret_cast<const uint4*>(a.v + ((size_t)b * a.Lk + j0 + jj) * a.ldv + h * DH + c * 8);
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

template <int DH>
__global__ void __launch_bounds__(T5_THREADS) t5_attn_fwd_kernel(T5AttnArgs a) {
    pdl_wait();
    a.drop.resolve();
    extern __shared__ float t5_smem[];
    float* Ks = t5_smem;                          // [64][DH + 1]
    float* Vs = Ks + T5_KEYS * (DH + 1);
    float* sbias = a.bias ? Vs + T5_KEYS * (DH + 1) : nullptr;   // [nb] this head's row of the table
    const int tid = threadIdx.x, r = tid >> 2, kq = tid & 3;
    const int b = blockIdx.y / a.H, h = blockIdx.y % a.H;
    const int i = blockIdx.x * T5_ROWS + r;
    if (sbias) for (int e = tid; e < a.nb; e += T5_THREADS) sbias[e] = a.bias[h * a.nb + e];
    float q[DH], o[DH];
#pragma unroll
    for (int d = 0; d < DH; ++d) { q[d] = 0.f; o[d] = 0.f; }
    if (i < a.Lq) t5_load_row<DH>(q, a.q + ((size_t)b * a.Lq + i) * a.ldq + h * DH);
    float m = -INFINITY, l = 0.f;
    const uint32_t drow = (uint32_t)(((size_t)b * a.H + h) * a.Lq + i);
    for (int j0 = 0; j0 < a.Lk; j0 += T5_KEYS) {
        __syncthreads();
        t5_load_tile<DH>(Ks, Vs, a, b, h, j0, tid);
        __syncthreads();
        if (i >= a.Lq) continue;
        for (int jj = kq; jj < T5_KEYS && j0 + jj < a.Lk; jj += 4) {
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
    if (i < a.Lq) {
        const float inv = l > 0.f ? __fdiv_rn(1.f, l) : 0.f;
        bf16* dst = a.out + ((size_t)b * a.Lq + i) * a.ldo + h * DH;
#pragma unroll
        for (int d = 0; d < DH; d += 2)
            if (((d >> 1) & 3) == kq) *reinterpret_cast<uint32_t*>(dst + d) = pack_bf16(o[d] * inv, o[d + 1] * inv);
        if (kq == 0) reinterpret_cast<float2*>(a.lse)[((size_t)b * a.H + h) * a.Lq + i] = make_float2(m, l);
    }
}

template <int DH>
__global__ void __launch_bounds__(T5_THREADS) t5_attn_bwd_kernel(T5AttnArgs a) {
    pdl_wait();
    a.drop.resolve();
    extern __shared__ float t5_smem[];
    float* Ks = t5_smem;                                  // [64][DH + 1]
    float* Vs = Ks + T5_KEYS * (DH + 1);
    float* Qs = Vs + T5_KEYS * (DH + 1);                  // [32][DH + 1]
    float* dOs = Qs + T5_ROWS * (DH + 1);                 // [32][DH + 1]
    float* dSs = dOs + T5_ROWS * (DH + 1);                // [32][64 + 1]  dS * scale (0 where not differentiable)
    float* Pds = dSs + T5_ROWS * (T5_KEYS + 1);           // [32][64 + 1]  dropped probabilities
    float* sbias = Pds + T5_ROWS * (T5_KEYS + 1);         // [nb]
    float* sdb = sbias + a.nb;                            // [nb] gradient bins of this CTA
    const int tid = threadIdx.x, r = tid >> 2, kq = tid & 3;
    const int b = blockIdx.y / a.H, h = blockIdx.y % a.H;
    const int i0 = blockIdx.x * T5_ROWS, i = i0 + r;
    const int D = a.H * DH;
    if (a.bias) for (int e = tid; e < a.nb; e += T5_THREADS) { sbias[e] = a.bias[h * a.nb + e]; sdb[e] = 0.f; }
    float q[DH], dO[DH], dq[DH];
#pragma unroll
    for (int d = 0; d < DH; ++d) { q[d] = 0.f; dO[d] = 0.f; dq[d] = 0.f; }
    float rmax = 0.f, rinv = 0.f, Dsum = 0.f;
    if (i < a.Lq) {
        t5_load_row<DH>(q, a.q + ((size_t)b * a.Lq + i) * a.ldq + h * DH);
        t5_load_row<DH>(dO, a.dout + ((size_t)b * a.Lq + i) * a.lddo + h * DH);
        float o[DH];
        t5_load_row<DH>(o, a.out + ((size_t)b * a.Lq + i) * a.ldo + h * DH);
#pragma unroll
        for (int d = 0; d < DH; ++d) Dsum = fmaf(dO[d], o[d], Dsum);   // rowsum(dO * O) = sum_j P_ij dP_ij
        const float2 ml = reinterpret_cast<const float2*>(a.lse)[((size_t)b * a.H + h) * a.Lq + i];
        rmax = ml.x; rinv = ml.y > 0.f ? __fdiv_rn(1.f, ml.y) : 0.f;
    }
    if (kq == 0) {
#pragma unroll
        for (int d = 0; d < DH; ++d) { Qs[r * (DH + 1) + d] = q[d]; dOs[r * (DH + 1) + d] = dO[d]; }
    }
    const uint32_t drow = (uint32_t)(((size_t)b * a.H + h) * a.Lq + i);
    for (int j0 = 0; j0 < a.Lk; j0 += T5_KEYS) {
        __syncthreads();
        t5_load_tile<DH>(Ks, Vs, a, b, h, j0, tid);
        for (int e = tid; e < T5_ROWS * (T5_KEYS + 1); e += T5_THREADS) { dSs[e] = 0.f; Pds[e] = 0.f; }
        __syncthreads();
        if (i < a.Lq) {
            for (int jj = kq; jj < T5_KEYS && j0 + jj < a.Lk; jj += 4) {
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
                    if (a.dbias) atomicAdd(&sdb[a.bucket[j0 + jj - i + a.Lq - 1]], ds);
                    const float dss = ds * a.scale;
                    dSs[r * (T5_KEYS + 1) + jj] = dss;
#pragma unroll
                    for (int d = 0; d < DH; ++d) dq[d] = fmaf(dss, kr[d], dq[d]);
                }
            }
        }
        __syncthreads();
        // dK_j += sum_r dS_rj q_r ; dV_j += sum_r Pd_rj dO_r : thread (key jj, half of the head dims), one atomic per (key, d)
        {
            const int jj = tid >> 1, half = tid & 1;
            if (j0 + jj < a.Lk) {
                float gk[DH / 2], gv[DH / 2];
#pragma unroll
                for (int d = 0; d < DH / 2; ++d) { gk[d] = 0.f; gv[d] = 0.f; }
                for (int rr = 0; rr < T5_ROWS; ++rr) {
                    const float ds = dSs[rr * (T5_KEYS + 1) + jj], pd = Pds[rr * (T5_KEYS + 1) + jj];
                    const float* qr = Qs + rr * (DH + 1) + half * (DH / 2);
                    const float* gr = dOs + rr * (DH + 1) + half * (DH / 2);
#pragma unroll
                    for (int d = 0; d < DH / 2; ++d) { gk[d] = fmaf(ds, qr[d], gk[d]); gv[d] = fmaf(pd, gr[d], gv[d]); }
                }
                float* dkp = a.dk + ((size_t)b * a.Lk + j0 + jj) * D + h * DH + half * (DH / 2);
                float* dvp = a.dv + ((size_t)b * a.Lk + j0 + jj) * D + h * DH + half * (DH / 2);
#pragma unroll
                for (int d = 0; d < DH / 2; ++d) { atomicAdd(dkp + d, gk[d]); atomicAdd(dvp + d, gv[d]); }
            }
        }
    }
#pragma unroll
    for (int d = 0; d < DH; ++d) {
        dq[d] += __shfl_xor_sync(0xffffffffu, dq[d], 1);
        dq[d] += __shfl_xor_sync(0xffffffffu, dq[d], 2);
    }
    if (i < a.Lq) {
        bf16* dst = a.dq + ((size_t)b * a.Lq + i) * a.lddq + h * DH;
#pragma unroll
        for (int d = 0; d < DH; d += 2)
            if (((d >> 1) & 3) == kq) *reinterpret_cast<uint32_t*>(dst + d) = pack_bf16(dq[d], dq[d + 1]);
    }
    if (a.dbias) {
        __syncthreads();
        for (int e = tid; e < a.nb; e += T5_THREADS)
            if (sdb[e] != 0.f) atomicAdd(a.dbias + h * a.nb + e, sdb[e]);
    }
}

template <int DH>
inline size_t t5_fwd_smem(int nb) { return (size_t)(2 * T5_KEYS * (DH + 1) + nb) * sizeof(float); }
template <int DH>
inline size_t t5_bwd_smem(int nb) {
    return (size_t)(2 * T5_KEYS * (DH + 1) + 2 * T5_ROWS * (DH + 1) + 2 * T5_ROWS * (T5_KEYS + 1) + 2 * nb) * sizeof(float);
}

}  // namespace grb
