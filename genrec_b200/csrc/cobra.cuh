// genrec_b200 - COBRA's item-text encoder and dense loss (genrec/models/cobra.py, genrec/modules/encoder.py:15-105).
//
//   packing     encoder_input_ids [N, L] -> token rows: text n is its leading non-zero tokens (none for a pad item), so neither the
//               pads of a text nor the texts of pad items are encoded.  Exact: the reference's key mask hides those keys, its pooling
//               hides those rows, and a text without tokens pools to zero whatever its rows hold.
//   pooling     pooled[n] = mean over the rows of text n of LayerNorm(row)                             (encoder.py:88-96)
//   l2norm      y = x / max(|x|, eps)                                                                  (F.normalize)
//   InfoNCE     loss_i = logsumexp_j(S_ij / tau) - S_ii / tau over the columns j outside [lo_i, hi_i), plus j = i   (cobra.py:484-493)
//
// Every cross-row sum runs in a fixed order (one CTA per text, warps in order; per-text partials added by det_finish), so two calls
// give the same bits.
#pragma once
#include "common.cuh"
#include "rowwise.cuh"   // LnStats, row_stats, ROW_THREADS
#include "tc_gemm.cuh"   // exp_accurate

namespace grb {

// ---- packing
// lens[n] = number of leading non-zero tokens of text n, 0 when keep[n] == 0, and -1 when a non-zero token follows a zero (a text
// that is not right-padded: the reference would attend to its later tokens, the packed rows could not).  One warp per text.
__global__ void __launch_bounds__(256) cobra_text_lens_kernel(const long long* __restrict__ tokens, int N, int L,
                                                             const unsigned char* __restrict__ keep, int* __restrict__ lens) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    for (long long n = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5; n < N; n += (long long)gridDim.x * 8) {
        const long long* t = tokens + n * L;
        int len = -1;          // first zero, -1 while none seen
        bool bad = false;
        for (int c = 0; c < L; c += 32) {
            const bool nz = c + lane < L && t[c + lane] != 0;
            const bool in = c + lane < L;
            const unsigned nzm = __ballot_sync(0xffffffffu, nz), zm = __ballot_sync(0xffffffffu, in && !nz);
            if (len >= 0) {
                bad |= nzm != 0u;
            } else if (zm) {
                const int z = __ffs(zm) - 1;
                len = c + z;
                bad |= (nzm >> z) != 0u;
            }
        }
        if (len < 0) len = L;
        if (lane == 0) lens[n] = (keep && !keep[n]) ? 0 : (bad ? -1 : len);
    }
}

// offsets[0 .. N] = exclusive scan of lens (a -1 counts as 0); info = {rows, longest text, first refused text + 1 or 0}.  One CTA.
constexpr int COBRA_SCAN_THREADS = 1024;
__global__ void __launch_bounds__(COBRA_SCAN_THREADS) cobra_text_offsets_kernel(const int* __restrict__ lens, int N,
                                                                               long long* __restrict__ offsets, long long* __restrict__ info) {
    pdl_wait();
    __shared__ long long wsum[32];
    __shared__ long long carry;
    __shared__ int longest, first_bad;
    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    if (tid == 0) { carry = 0; longest = 0; first_bad = INT_MAX; offsets[0] = 0; }
    __syncthreads();
    for (int base = 0; base < N; base += COBRA_SCAN_THREADS) {
        const int n = base + tid;
        const int raw = n < N ? lens[n] : 0;
        if (raw < 0) atomicMin(&first_bad, n);
        const long long v = raw > 0 ? raw : 0;
        if (v > 0) atomicMax(&longest, (int)v);
        long long incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long u = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += u;
        }
        if (lane == 31) wsum[w] = incl;
        __syncthreads();
        if (w == 0) {
            long long s = wsum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const long long u = __shfl_up_sync(0xffffffffu, s, o);
                if (lane >= o) s += u;
            }
            wsum[lane] = s;
        }
        __syncthreads();
        const long long before = carry + (w > 0 ? wsum[w - 1] : 0);
        if (n < N) offsets[n + 1] = before + incl;
        __syncthreads();
        if (tid == 0) carry += wsum[31];
        __syncthreads();
    }
    if (tid == 0) {
        info[0] = carry;
        info[1] = longest;
        info[2] = first_bad == INT_MAX ? 0 : (long long)first_bad + 1;
    }
}

// rows of text n: tok[offsets[n] + l] = tokens[n, l], pos[...] = l for l < len.  One warp per text.
__global__ void __launch_bounds__(256) cobra_text_rows_kernel(const long long* __restrict__ tokens, int N, int L,
                                                             const long long* __restrict__ offsets, long long* __restrict__ tok,
                                                             long long* __restrict__ pos) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    for (long long n = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5; n < N; n += (long long)gridDim.x * 8) {
        const long long r0 = offsets[n];
        const int len = (int)(offsets[n + 1] - r0);
        for (int l = lane; l < len; l += 32) {
            tok[r0 + l] = tokens[n * L + l];
            pos[r0 + l] = l;
        }
    }
}

// ---- pooling: one CTA (8 warps) per text; warp w takes rows w, w + 8, ... of it.  D = 64 NP.
struct SegLnArgs {
    const long long* offsets;   // [N + 1] row offsets of the texts
    int N, D;
    float eps;
    const float* x;             // [rows, D] the encoder's output rows
    const float *g, *b;         // LayerNorm weight / bias [D]
    float* st;                  // [rows, 2] {mean, rstd}
    float* pooled;              // [N, D] (forward)
    const float* dpooled;       // [N, D] (backward)
    float* dx;                  // [rows, D] (backward)
    float* part;                // [2][N][D] per-text dg / db (backward; det_finish adds them)
};
template <int NP>
__global__ void __launch_bounds__(ROW_THREADS) seg_ln_mean_fwd_kernel(SegLnArgs a) {
    pdl_wait();
    __shared__ float red[ROW_THREADS / 32][64 * NP];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, n = blockIdx.x;
    const long long r0 = a.offsets[n];
    const int len = (int)(a.offsets[n + 1] - r0);
    float acc[NP][2];
#pragma unroll
    for (int p = 0; p < NP; ++p) acc[p][0] = acc[p][1] = 0.f;
    for (int r = w; r < len; r += ROW_THREADS / 32) {
        const size_t row = (size_t)(r0 + r);
        float xv[NP][2];
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            const float2 f = *reinterpret_cast<const float2*>(a.x + row * a.D + 2 * lane + 64 * p);
            xv[p][0] = f.x; xv[p][1] = f.y;
        }
        const LnStats s = row_stats<NP>(xv, a.D, a.eps);
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            const int c = 2 * lane + 64 * p;
            acc[p][0] += (xv[p][0] - s.mean) * s.rstd * a.g[c] + a.b[c];
            acc[p][1] += (xv[p][1] - s.mean) * s.rstd * a.g[c + 1] + a.b[c + 1];
        }
        if (lane == 0) { a.st[2 * row] = s.mean; a.st[2 * row + 1] = s.rstd; }
    }
#pragma unroll
    for (int p = 0; p < NP; ++p) { red[w][2 * lane + 64 * p] = acc[p][0]; red[w][2 * lane + 64 * p + 1] = acc[p][1]; }
    __syncthreads();
    const float cnt = (float)(len > 0 ? len : 1);
    for (int c = threadIdx.x; c < a.D; c += ROW_THREADS) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < ROW_THREADS / 32; ++k) s += red[k][c];
        a.pooled[(size_t)n * a.D + c] = __fdiv_rn(s, cnt);
    }
}
// dx = LNbwd(dpooled[n] / len) for each row of text n; the text's dg / db go to part[0 / 1][n]
template <int NP>
__global__ void __launch_bounds__(ROW_THREADS) seg_ln_mean_bwd_kernel(SegLnArgs a) {
    pdl_wait();
    __shared__ float red[ROW_THREADS / 32][64 * NP];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, n = blockIdx.x;
    const long long r0 = a.offsets[n];
    const int len = (int)(a.offsets[n + 1] - r0);
    const float cnt = (float)(len > 0 ? len : 1), invD = 1.f / (float)a.D;
    float dy[NP][2], adg[NP][2];
#pragma unroll
    for (int p = 0; p < NP; ++p) {
        const float2 f = *reinterpret_cast<const float2*>(a.dpooled + (size_t)n * a.D + 2 * lane + 64 * p);
        dy[p][0] = __fdiv_rn(f.x, cnt); dy[p][1] = __fdiv_rn(f.y, cnt);
        adg[p][0] = adg[p][1] = 0.f;
    }
    for (int r = w; r < len; r += ROW_THREADS / 32) {
        const size_t row = (size_t)(r0 + r);
        const float m = a.st[2 * row], rs = a.st[2 * row + 1];
        float xh[NP][2], gg[NP][2], sa = 0.f, sb = 0.f;
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            const int c = 2 * lane + 64 * p;
            const float2 xv = *reinterpret_cast<const float2*>(a.x + row * a.D + c);
            xh[p][0] = (xv.x - m) * rs; xh[p][1] = (xv.y - m) * rs;
            adg[p][0] += dy[p][0] * xh[p][0]; adg[p][1] += dy[p][1] * xh[p][1];
            gg[p][0] = dy[p][0] * a.g[c]; gg[p][1] = dy[p][1] * a.g[c + 1];
            sa += gg[p][0] + gg[p][1];
            sb += gg[p][0] * xh[p][0] + gg[p][1] * xh[p][1];
        }
        sa = warp_sum(sa) * invD; sb = warp_sum(sb) * invD;
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            const int c = 2 * lane + 64 * p;
            *reinterpret_cast<float2*>(a.dx + row * a.D + c) =
                make_float2(rs * (gg[p][0] - sa - xh[p][0] * sb), rs * (gg[p][1] - sa - xh[p][1] * sb));
        }
    }
#pragma unroll
    for (int p = 0; p < NP; ++p) { red[w][2 * lane + 64 * p] = adg[p][0]; red[w][2 * lane + 64 * p + 1] = adg[p][1]; }
    __syncthreads();
    det_store(a.part, 0, n, a.N, a.D, a.D, [&](int c) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < ROW_THREADS / 32; ++k) s += red[k][c];
        return s;
    });
    // every row of the text has the same dy: its db is len * dy
    det_store(a.part, 1, n, a.N, a.D, a.D, [&](int c) { return __fdiv_rn(a.dpooled[(size_t)n * a.D + c], cnt) * (float)len; });
}

// ---- L2 normalisation, one warp per row (D % 32 == 0, D <= 1024)
__global__ void __launch_bounds__(256) l2norm_fwd_kernel(const float* __restrict__ x, int T, int D, float eps, float* __restrict__ y,
                                                        float* __restrict__ nrm) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    for (long long row = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5; row < T; row += (long long)gridDim.x * 8) {
        const float* xr = x + row * D;
        float s = 0.f;
        for (int c = lane; c < D; c += 32) s = fmaf(xr[c], xr[c], s);
        const float n = sqrtf(warp_sum(s)), d = fmaxf(n, eps);
        for (int c = lane; c < D; c += 32) y[row * D + c] = __fdiv_rn(xr[c], d);
        if (lane == 0 && nrm) nrm[row] = n;
    }
}
// dx = (dy - y (dy . y)) / |x| where |x| > eps, else dy / eps (the clamp passes no gradient to the norm)
__global__ void __launch_bounds__(256) l2norm_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y,
                                                        const float* __restrict__ nrm, int T, int D, float eps, float* __restrict__ dx) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    for (long long row = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5; row < T; row += (long long)gridDim.x * 8) {
        const float n = nrm[row];
        const float* g = dy + row * D;
        const float* yr = y + row * D;
        if (n > eps) {
            float s = 0.f;
            for (int c = lane; c < D; c += 32) s = fmaf(g[c], yr[c], s);
            s = warp_sum(s);
            for (int c = lane; c < D; c += 32) dx[row * D + c] = __fdiv_rn(g[c] - yr[c] * s, n);
        } else {
            for (int c = lane; c < D; c += 32) dx[row * D + c] = __fdiv_rn(g[c], eps);
        }
    }
}

// ---- InfoNCE rows.  S [Q, ld] fp32 scores pred . gt (columns [Q, ld) are padding); row i leaves out the columns [lo[i], hi[i])
// except i itself (the other items of its own sequence, which the reference fills with -1e4: exp(-1e4 - max) is 0 in fp32).
// row_loss[i] = lse_i - S_ii / tau ; dS[i, j] = bf16((softmax_ij - [i == j]) / (Q tau)), 0 in the left-out and padding columns.
// One CTA per row.
__global__ void __launch_bounds__(256) infonce_rows_kernel(const float* __restrict__ S, int Q, int ld, const long long* __restrict__ lo,
                                                          const long long* __restrict__ hi, float inv_tau, float* __restrict__ row_loss,
                                                          bf16* __restrict__ dS) {
    pdl_wait();
    __shared__ float red[8];
    __shared__ float bcast;
    const int i = blockIdx.x, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const float* s = S + (size_t)i * ld;
    const long long l0 = lo[i], l1 = hi[i];
    auto keep = [&](int j) { return j == i || j < l0 || j >= l1; };
    // every use of a logit rounds it once, the same way (no product fused into the subtraction that follows): the row's own logit
    // minus the max is then exactly 0 where the row keeps only itself, whose loss is exactly 0
    auto logit = [&](int j) { return __fmul_rn(s[j], inv_tau); };
    float m = -INFINITY;
    for (int j = tid; j < Q; j += 256)
        if (keep(j)) m = fmaxf(m, logit(j));
    m = warp_max(m);
    if (lane == 0) red[w] = m;
    __syncthreads();
    if (tid == 0) {
        float v = red[0];
        for (int k = 1; k < 8; ++k) v = fmaxf(v, red[k]);
        bcast = v;
    }
    __syncthreads();
    m = bcast;
    float z = 0.f;
    for (int j = tid; j < Q; j += 256)
        if (keep(j)) z += exp_accurate(logit(j) - m);
    z = warp_sum(z);
    __syncthreads();
    if (lane == 0) red[w] = z;
    __syncthreads();
    if (tid == 0) {
        float v = 0.f;
        for (int k = 0; k < 8; ++k) v += red[k];
        bcast = v;
        row_loss[i] = logf(v) + (m - logit(i));
    }
    __syncthreads();
    const float inv_z = __fdiv_rn(1.f, bcast), gscale = __fdiv_rn(inv_tau, (float)Q);
    bf16* d = dS + (size_t)i * ld;
    for (int j = tid; j < ld; j += 256) {
        float g = 0.f;
        if (j < Q && keep(j)) g = (exp_accurate(logit(j) - m) * inv_z - (j == i ? 1.f : 0.f)) * gscale;
        d[j] = __float2bfloat16_rn(g);
    }
}

}  // namespace grb
