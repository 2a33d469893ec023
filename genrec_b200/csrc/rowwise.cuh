// genrec_b200 - row-wise (per token) kernels: LayerNorm / gate / residual forward+backward, casts, column sums,
// embedding gather/scatter, cross-entropy over bf16 logits, fused Adam.  HBM-bound; one warp per token row,
// 8-byte (bf16x4 / float2) vector accesses, D % 64 == 0, D <= 512.
#pragma once
#include "common.cuh"

namespace grb {

constexpr int ROW_THREADS = 256;  // 8 warps = 8 rows in flight per CTA

struct LnStats { float mean, rstd; };

// lane owns column pairs c = 2*lane + 64*p , p < NP
template <int NP>
GRB_DEVINL LnStats row_stats(const float (&v)[NP][2], int D, float eps) {
    float s = 0.f;
#pragma unroll
    for (int p = 0; p < NP; ++p) s += v[p][0] + v[p][1];
    float mean = warp_sum(s) / (float)D;
    float q = 0.f;
#pragma unroll
    for (int p = 0; p < NP; ++p) {
        float a = v[p][0] - mean, b = v[p][1] - mean;
        q += a * a + b * b;
    }
    float var = warp_sum(q) / (float)D;
    LnStats st;
    st.mean = mean;
    st.rstd = rsqrtf(var + eps);
    return st;
}

// ------------------------------------------------------------------------------------------------ HSTU: norm + gate + residual + norm
//   N = LN1(O) ; x1 = x + drop(N * U) ; xn = LN2(x1)          (genrec/models/hstu.py:271-278)
struct LnGateFwdArgs {
    const bf16* O; int ldo;
    const bf16* U; int ldu;
    const float* x;
    const float *g1, *b1, *g2, *b2;
    float* x1; bf16* xn;
    float* st1; float* st2;  // [T,2]
    int T, D;
    float eps;
    Dropout drop;
};
template <int NP>
__global__ void __launch_bounds__(ROW_THREADS) ln_gate_fwd_kernel(LnGateFwdArgs a) {
    pdl_wait();
    a.drop.resolve();
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nw = gridDim.x * (ROW_THREADS / 32);
    for (int row = blockIdx.x * (ROW_THREADS / 32) + wib; row < a.T; row += nw) {
        float o[NP][2], u[NP][2], xv[NP][2];
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            int c = 2 * lane + 64 * p;
            float2 t = unpack_bf16(*reinterpret_cast<const uint32_t*>(a.O + (size_t)row * a.ldo + c));
            o[p][0] = t.x; o[p][1] = t.y;
            t = unpack_bf16(*reinterpret_cast<const uint32_t*>(a.U + (size_t)row * a.ldu + c));
            u[p][0] = t.x; u[p][1] = t.y;
            float2 f = *reinterpret_cast<const float2*>(a.x + (size_t)row * a.D + c);
            xv[p][0] = f.x; xv[p][1] = f.y;
        }
        LnStats s1 = row_stats<NP>(o, a.D, a.eps);
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            int c = 2 * lane + 64 * p;
            float gv[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) gv[e] = ((o[p][e] - s1.mean) * s1.rstd * a.g1[c + e] + a.b1[c + e]) * u[p][e];
            a.drop.apply2(gv[0], gv[1], row, c);
            xv[p][0] += gv[0];
            xv[p][1] += gv[1];
            *reinterpret_cast<float2*>(a.x1 + (size_t)row * a.D + c) = make_float2(xv[p][0], xv[p][1]);
        }
        LnStats s2 = row_stats<NP>(xv, a.D, a.eps);
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            int c = 2 * lane + 64 * p;
            float y0 = (xv[p][0] - s2.mean) * s2.rstd * a.g2[c] + a.b2[c];
            float y1 = (xv[p][1] - s2.mean) * s2.rstd * a.g2[c + 1] + a.b2[c + 1];
            *reinterpret_cast<uint32_t*>(a.xn + (size_t)row * a.D + c) = pack_bf16(y0, y1);
        }
        if (lane == 0) {
            a.st1[2 * row] = s1.mean; a.st1[2 * row + 1] = s1.rstd;
            a.st2[2 * row] = s2.mean; a.st2[2 * row + 1] = s2.rstd;
        }
    }
}

// backward of the above.  dy: grad of the layer output (flows through the FFN residual), dxn: grad of LN2 output.
struct LnGateBwdArgs {
    const float* dy; const float* dxn;
    const float* x1; const float* st1; const float* st2;
    const bf16* O; int ldo;
    const bf16* U; int ldu;
    const bf16* zu; int ldz;       // pre-activation of U (for silu')
    const float *g1, *b1, *g2;
    float* dx1;                    // [T,D] fp32
    bf16* dO; int lddo;            // [T,D]
    bf16* dzu; int lddz;           // [T, ...] grad wrt U pre-activation
    float *dg1, *db1, *dg2, *db2;  // accumulated
    int T, D;
    Dropout drop;
    float* part;                   // [4][gridDim.x][D] scratch for the ordered cross-CTA sum (det_finish_kernel)
};
template <int NP>
__global__ void __launch_bounds__(ROW_THREADS) ln_gate_bwd_kernel(LnGateBwdArgs a) {
    pdl_wait();
    a.drop.resolve();
    __shared__ float red[4][ROW_THREADS / 32][64 * NP];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nw = gridDim.x * (ROW_THREADS / 32);
    float adg1[NP][2], adb1[NP][2], adg2[NP][2], adb2[NP][2];
#pragma unroll
    for (int p = 0; p < NP; ++p)
#pragma unroll
        for (int e = 0; e < 2; ++e) adg1[p][e] = adb1[p][e] = adg2[p][e] = adb2[p][e] = 0.f;
    const float invD = 1.f / (float)a.D;

    for (int row = blockIdx.x * (ROW_THREADS / 32) + wib; row < a.T; row += nw) {
        const float m1 = a.st1[2 * row], r1 = a.st1[2 * row + 1], m2 = a.st2[2 * row], r2 = a.st2[2 * row + 1];
        // every operand of the row is requested up front (one memory round trip instead of two dependent phases)
        float2 xv[NP], dn[NP], dyv[NP];
        uint32_t ovp[NP], uvp[NP], zvp[NP];
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            const int c = 2 * lane + 64 * p;
            xv[p] = *reinterpret_cast<const float2*>(a.x1 + (size_t)row * a.D + c);
            dn[p] = *reinterpret_cast<const float2*>(a.dxn + (size_t)row * a.D + c);
            dyv[p] = *reinterpret_cast<const float2*>(a.dy + (size_t)row * a.D + c);
            ovp[p] = *reinterpret_cast<const uint32_t*>(a.O + (size_t)row * a.ldo + c);
            uvp[p] = *reinterpret_cast<const uint32_t*>(a.U + (size_t)row * a.ldu + c);
            zvp[p] = *reinterpret_cast<const uint32_t*>(a.zu + (size_t)row * a.ldz + c);
        }
        float xh2[NP][2], gg[NP][2], dx1[NP][2];
        float sa = 0.f, sb = 0.f;
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            int c = 2 * lane + 64 * p;
            xh2[p][0] = (xv[p].x - m2) * r2; xh2[p][1] = (xv[p].y - m2) * r2;
            adg2[p][0] += dn[p].x * xh2[p][0]; adg2[p][1] += dn[p].y * xh2[p][1];
            adb2[p][0] += dn[p].x; adb2[p][1] += dn[p].y;
            gg[p][0] = dn[p].x * a.g2[c]; gg[p][1] = dn[p].y * a.g2[c + 1];
            sa += gg[p][0] + gg[p][1];
            sb += gg[p][0] * xh2[p][0] + gg[p][1] * xh2[p][1];
        }
        sa = warp_sum(sa) * invD; sb = warp_sum(sb) * invD;
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            int c = 2 * lane + 64 * p;
            dx1[p][0] = dyv[p].x + r2 * (gg[p][0] - sa - xh2[p][0] * sb);
            dx1[p][1] = dyv[p].y + r2 * (gg[p][1] - sa - xh2[p][1] * sb);
            *reinterpret_cast<float2*>(a.dx1 + (size_t)row * a.D + c) = make_float2(dx1[p][0], dx1[p][1]);
        }
        // gate + LN1
        float xh1[NP][2], gn[NP][2];
        float ta = 0.f, tb = 0.f;
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            int c = 2 * lane + 64 * p;
            float2 ov = unpack_bf16(ovp[p]);
            float2 uv = unpack_bf16(uvp[p]);
            float2 zv = unpack_bf16(zvp[p]);
            float o2[2] = {ov.x, ov.y}, u2[2] = {uv.x, uv.y}, z2[2] = {zv.x, zv.y}, dzu[2];
            float dGv[2] = {dx1[p][0], dx1[p][1]};
            a.drop.apply2(dGv[0], dGv[1], row, c);
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const float dG = dGv[e];
                xh1[p][e] = (o2[e] - m1) * r1;
                float n = xh1[p][e] * a.g1[c + e] + a.b1[c + e];
                dzu[e] = dG * n * dsiluf(z2[e]);
                float dN = dG * u2[e];
                adg1[p][e] += dN * xh1[p][e];
                adb1[p][e] += dN;
                gn[p][e] = dN * a.g1[c + e];
                ta += gn[p][e];
                tb += gn[p][e] * xh1[p][e];
            }
            *reinterpret_cast<uint32_t*>(a.dzu + (size_t)row * a.lddz + c) = pack_bf16(dzu[0], dzu[1]);
        }
        ta = warp_sum(ta) * invD; tb = warp_sum(tb) * invD;
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            int c = 2 * lane + 64 * p;
            float d0 = r1 * (gn[p][0] - ta - xh1[p][0] * tb), d1 = r1 * (gn[p][1] - ta - xh1[p][1] * tb);
            *reinterpret_cast<uint32_t*>(a.dO + (size_t)row * a.lddo + c) = pack_bf16(d0, d1);
        }
    }
    // CTA reduction of the four parameter-gradient vectors, then the ordered cross-CTA sum
#pragma unroll
    for (int p = 0; p < NP; ++p)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            int c = 2 * lane + 64 * p + e;
            red[0][wib][c] = adg1[p][e]; red[1][wib][c] = adb1[p][e];
            red[2][wib][c] = adg2[p][e]; red[3][wib][c] = adb2[p][e];
        }
    __syncthreads();
    for (int which = 0; which < 4; ++which) {
        auto colsum = [&](int c) {
            float s = 0.f;
#pragma unroll
            for (int w = 0; w < ROW_THREADS / 32; ++w) s += red[which][w][c];
            return s;
        };
        det_store(a.part, which, blockIdx.x, gridDim.x, a.D, a.D, colsum);
    }
}

// ------------------------------------------------------------------------------------------------ plain LayerNorm fwd / bwd
// y = LN(x) (fp32 in) -> bf16 and/or fp32 out, stats saved.
struct LnFwdArgs {
    const float* x; const float *g, *b;
    bf16* y_bf16; float* y_f32;  // either nullable
    float* st;
    int T, D; float eps;
};
template <int NP>
__global__ void __launch_bounds__(ROW_THREADS) ln_fwd_kernel(LnFwdArgs a) {
    pdl_wait();
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nw = gridDim.x * (ROW_THREADS / 32);
    for (int row = blockIdx.x * (ROW_THREADS / 32) + wib; row < a.T; row += nw) {
        float xv[NP][2];
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            float2 f = *reinterpret_cast<const float2*>(a.x + (size_t)row * a.D + 2 * lane + 64 * p);
            xv[p][0] = f.x; xv[p][1] = f.y;
        }
        LnStats s = row_stats<NP>(xv, a.D, a.eps);
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            int c = 2 * lane + 64 * p;
            float y0 = (xv[p][0] - s.mean) * s.rstd * a.g[c] + a.b[c];
            float y1 = (xv[p][1] - s.mean) * s.rstd * a.g[c + 1] + a.b[c + 1];
            if (a.y_bf16) *reinterpret_cast<uint32_t*>(a.y_bf16 + (size_t)row * a.D + c) = pack_bf16(y0, y1);
            if (a.y_f32) *reinterpret_cast<float2*>(a.y_f32 + (size_t)row * a.D + c) = make_float2(y0, y1);
        }
        if (lane == 0 && a.st) { a.st[2 * row] = s.mean; a.st[2 * row + 1] = s.rstd; }
    }
}
// dx = (res ? res : 0) + LNbwd(dy) ; dg += , db +=
struct LnBwdArgs {
    const float* dy; const float* x; const float* st; const float* g;
    const float* res;  // nullable, added to dx
    float* dx; float *dg, *db;
    int T, D;
    float* part;       // [2][gridDim.x][D] scratch for the ordered cross-CTA sum (det_finish_kernel adds it to dg, db)
};
template <int NP>
__global__ void __launch_bounds__(ROW_THREADS) ln_bwd_kernel(LnBwdArgs a) {
    pdl_wait();
    __shared__ float red[2][ROW_THREADS / 32][64 * NP];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nw = gridDim.x * (ROW_THREADS / 32);
    float adg[NP][2], adb[NP][2];
#pragma unroll
    for (int p = 0; p < NP; ++p) adg[p][0] = adg[p][1] = adb[p][0] = adb[p][1] = 0.f;
    const float invD = 1.f / (float)a.D;
    for (int row = blockIdx.x * (ROW_THREADS / 32) + wib; row < a.T; row += nw) {
        const float m = a.st[2 * row], r = a.st[2 * row + 1];
        float xh[NP][2], gg[NP][2];
        float sa = 0.f, sb = 0.f;
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            int c = 2 * lane + 64 * p;
            float2 xv = *reinterpret_cast<const float2*>(a.x + (size_t)row * a.D + c);
            float2 dv = *reinterpret_cast<const float2*>(a.dy + (size_t)row * a.D + c);
            xh[p][0] = (xv.x - m) * r; xh[p][1] = (xv.y - m) * r;
            adg[p][0] += dv.x * xh[p][0]; adg[p][1] += dv.y * xh[p][1];
            adb[p][0] += dv.x; adb[p][1] += dv.y;
            gg[p][0] = dv.x * a.g[c]; gg[p][1] = dv.y * a.g[c + 1];
            sa += gg[p][0] + gg[p][1];
            sb += gg[p][0] * xh[p][0] + gg[p][1] * xh[p][1];
        }
        sa = warp_sum(sa) * invD; sb = warp_sum(sb) * invD;
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            int c = 2 * lane + 64 * p;
            float d0 = r * (gg[p][0] - sa - xh[p][0] * sb), d1 = r * (gg[p][1] - sa - xh[p][1] * sb);
            if (a.res) {
                float2 rv = *reinterpret_cast<const float2*>(a.res + (size_t)row * a.D + c);
                d0 += rv.x; d1 += rv.y;
            }
            *reinterpret_cast<float2*>(a.dx + (size_t)row * a.D + c) = make_float2(d0, d1);
        }
    }
#pragma unroll
    for (int p = 0; p < NP; ++p)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            int c = 2 * lane + 64 * p + e;
            red[0][wib][c] = adg[p][e]; red[1][wib][c] = adb[p][e];
        }
    __syncthreads();
    for (int which = 0; which < 2; ++which) {
        auto colsum = [&](int c) {
            float s = 0.f;
#pragma unroll
            for (int w = 0; w < ROW_THREADS / 32; ++w) s += red[which][w][c];
            return s;
        };
        det_store(a.part, which, blockIdx.x, gridDim.x, a.D, a.D, colsum);
    }
}

// ------------------------------------------------------------------------------------------------ T5 RMS norm fwd / bwd
// y = w * (x * r), r = rsqrt(mean(x^2) + eps)   (genrec/modules/normalize.py:38-55 and :73-96: no mean, no bias)
struct RmsFwdArgs {
    const float* x; const float* w;
    bf16* y_bf16; float* y_f32;  // either nullable
    float* rstd;                 // nullable [T]
    int T, D; float eps;
};
template <int NP>
__global__ void __launch_bounds__(ROW_THREADS) rms_fwd_kernel(RmsFwdArgs a) {
    pdl_wait();
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nw = gridDim.x * (ROW_THREADS / 32);
    for (int row = blockIdx.x * (ROW_THREADS / 32) + wib; row < a.T; row += nw) {
        float xv[NP][2];
        float q = 0.f;
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            float2 f = *reinterpret_cast<const float2*>(a.x + (size_t)row * a.D + 2 * lane + 64 * p);
            xv[p][0] = f.x; xv[p][1] = f.y;
            q += f.x * f.x + f.y * f.y;
        }
        const float r = rsqrtf(warp_sum(q) / (float)a.D + a.eps);
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            int c = 2 * lane + 64 * p;
            float y0 = a.w[c] * (xv[p][0] * r), y1 = a.w[c + 1] * (xv[p][1] * r);
            if (a.y_bf16) *reinterpret_cast<uint32_t*>(a.y_bf16 + (size_t)row * a.D + c) = pack_bf16(y0, y1);
            if (a.y_f32) *reinterpret_cast<float2*>(a.y_f32 + (size_t)row * a.D + c) = make_float2(y0, y1);
        }
        if (lane == 0 && a.rstd) a.rstd[row] = r;
    }
}
// dx = (res ? res : 0) + r * (g - xh * mean(g * xh)), g = dy * w, xh = x * r ; dw += sum over rows of dy * xh
struct RmsBwdArgs {
    const float* dy; const float* x; const float* rstd; const float* w;
    const float* res;  // nullable, added to dx
    float* dx; float* dw;
    int T, D;
    float* part;       // [gridDim.x][D] scratch for the ordered cross-CTA sum (det_finish_kernel adds it to dw)
};
template <int NP>
__global__ void __launch_bounds__(ROW_THREADS) rms_bwd_kernel(RmsBwdArgs a) {
    pdl_wait();
    __shared__ float red[ROW_THREADS / 32][64 * NP];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nw = gridDim.x * (ROW_THREADS / 32);
    float adw[NP][2];
#pragma unroll
    for (int p = 0; p < NP; ++p) adw[p][0] = adw[p][1] = 0.f;
    const float invD = 1.f / (float)a.D;
    for (int row = blockIdx.x * (ROW_THREADS / 32) + wib; row < a.T; row += nw) {
        const float r = a.rstd[row];
        float xh[NP][2], gg[NP][2];
        float sb = 0.f;
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            int c = 2 * lane + 64 * p;
            float2 xv = *reinterpret_cast<const float2*>(a.x + (size_t)row * a.D + c);
            float2 dv = *reinterpret_cast<const float2*>(a.dy + (size_t)row * a.D + c);
            xh[p][0] = xv.x * r; xh[p][1] = xv.y * r;
            adw[p][0] += dv.x * xh[p][0]; adw[p][1] += dv.y * xh[p][1];
            gg[p][0] = dv.x * a.w[c]; gg[p][1] = dv.y * a.w[c + 1];
            sb += gg[p][0] * xh[p][0] + gg[p][1] * xh[p][1];
        }
        sb = warp_sum(sb) * invD;
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            int c = 2 * lane + 64 * p;
            float d0 = r * (gg[p][0] - xh[p][0] * sb), d1 = r * (gg[p][1] - xh[p][1] * sb);
            if (a.res) {
                float2 rv = *reinterpret_cast<const float2*>(a.res + (size_t)row * a.D + c);
                d0 += rv.x; d1 += rv.y;
            }
            *reinterpret_cast<float2*>(a.dx + (size_t)row * a.D + c) = make_float2(d0, d1);
        }
    }
#pragma unroll
    for (int p = 0; p < NP; ++p)
#pragma unroll
        for (int e = 0; e < 2; ++e) red[wib][2 * lane + 64 * p + e] = adw[p][e];
    __syncthreads();
    auto colsum = [&](int c) {
        float s = 0.f;
#pragma unroll
        for (int w = 0; w < ROW_THREADS / 32; ++w) s += red[w][c];
        return s;
    };
    det_store(a.part, 0, blockIdx.x, gridDim.x, a.D, a.D, colsum);
}

// ------------------------------------------------------------------------------------------------ casts / column sums
// out_bf16[i] = bf16(dropmask(in[i]) * row_scale[row])       (n = T*D elements, D = row length)
__global__ void cast_f32_bf16_kernel(const float* __restrict__ in, bf16* __restrict__ out, size_t n, int D, Dropout drop,
                                     const float* __restrict__ row_scale) {
    pdl_wait();
    drop.resolve();
    // a thread converts 4 neighbouring columns per step; (row, column) advance without divisions inside the loop
    const size_t nq = n / 4, stride = (size_t)gridDim.x * blockDim.x;
    const uint32_t D4 = (uint32_t)D / 4;
    size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;   // < 2^32 (the grid is capped), as is stride
    uint32_t row = (uint32_t)q / D4, cq = (uint32_t)q % D4;
    const uint32_t srow = (uint32_t)stride / D4, scq = (uint32_t)stride % D4;
    for (; q < nq; q += stride) {
        const size_t i = q * 4;
        float4 v = *reinterpret_cast<const float4*>(in + i);
        const float rs = row_scale ? row_scale[row] : 1.f;
        uint2 o;
        drop.apply2(v.x, v.y, row, cq * 4);
        drop.apply2(v.z, v.w, row, cq * 4 + 2);
        o.x = pack_bf16(v.x * rs, v.y * rs);
        o.y = pack_bf16(v.z * rs, v.w * rs);
        *reinterpret_cast<uint2*>(out + i) = o;
        row += srow;
        cq += scq;
        if (cq >= D4) { cq -= D4; ++row; }
    }
}
// out_bf16[r, c] = bf16(dropmask(in[r, c]))  and  the per-CTA column sums of out_bf16 -> part [ceil(D / 128)][chunks][128], which
// det_finish_kernel adds to the bias gradient (the cast of dy and the bias gradient of the layer's last linear in one pass).
// grid (ceil(D / 128), chunks) ; block 256 = 8 row lanes x 32 threads of 4 columns.
__global__ void __launch_bounds__(256) cast_colsum_f32_bf16_kernel(const float* __restrict__ in, bf16* __restrict__ out, int T, int D,
                                                                  Dropout drop, float* __restrict__ part) {
    pdl_wait();
    drop.resolve();
    __shared__ float red[8][128];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int c = blockIdx.x * 128 + 4 * tx;
    const int rows_per = (T + gridDim.y - 1) / gridDim.y;
    const int r0 = blockIdx.y * rows_per, r1 = min(T, r0 + rows_per);
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    if (c < D) {
        auto one = [&](int r, float4 v) {
            drop.apply2(v.x, v.y, r, c);
            drop.apply2(v.z, v.w, r, c + 2);
            uint2 o;
            o.x = pack_bf16(v.x, v.y);
            o.y = pack_bf16(v.z, v.w);
            *reinterpret_cast<uint2*>(out + (size_t)r * D + c) = o;
            const float2 a = unpack_bf16(o.x), b = unpack_bf16(o.y);
            s[0] += a.x; s[1] += a.y; s[2] += b.x; s[3] += b.y;
        };
        int r = r0 + ty;
        for (; r + 24 < r1; r += 32) {
            float4 q[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) q[u] = *reinterpret_cast<const float4*>(in + (size_t)(r + 8 * u) * D + c);
#pragma unroll
            for (int u = 0; u < 4; ++u) one(r + 8 * u, q[u]);
        }
        for (; r < r1; r += 8) one(r, *reinterpret_cast<const float4*>(in + (size_t)r * D + c));
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) red[ty][4 * tx + k] = s[k];
    __syncthreads();
    auto sum8 = [&](int i) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += red[w][i];
        return t;
    };
    det_store(part, blockIdx.x, blockIdx.y, gridDim.y, 128, min(128, D - (int)blockIdx.x * 128), sum8);
}
// the per-CTA column sums of in: bf16 [T, ld] (ld % 8 == 0), columns [0, N) -> part [ceil(N / 256)][chunks][256], which
// det_finish_kernel adds to the output ; grid (ceil(N/256), chunks) ;
// block 256 = 32 column groups of 8 (one 16-byte load each) x 8 row lanes, 4 rows in flight per thread
__global__ void __launch_bounds__(256) colsum_bf16_kernel(const bf16* __restrict__ in, int T, int N, int ld, float* __restrict__ part) {
    pdl_wait();
    __shared__ float red[8][256];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int c = blockIdx.x * 256 + 8 * tx;
    const int rows_per = (T + gridDim.y - 1) / gridDim.y;
    const int r0 = blockIdx.y * rows_per, r1 = min(T, r0 + rows_per);
    float s[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) s[k] = 0.f;
    if (c < N) {
        int r = r0 + ty;
        for (; r + 24 < r1; r += 32) {
            uint4 q[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) q[u] = *reinterpret_cast<const uint4*>(in + (size_t)(r + 8 * u) * ld + c);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const uint32_t w[4] = {q[u].x, q[u].y, q[u].z, q[u].w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    float2 f = unpack_bf16(w[k]);
                    s[2 * k] += f.x; s[2 * k + 1] += f.y;
                }
            }
        }
        for (; r < r1; r += 8) {
            const uint4 q = *reinterpret_cast<const uint4*>(in + (size_t)r * ld + c);
            const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float2 f = unpack_bf16(w[k]);
                s[2 * k] += f.x; s[2 * k + 1] += f.y;
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) red[ty][8 * tx + k] = s[k];
    __syncthreads();
    auto sum8 = [&](int i) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += red[w][i];
        return t;
    };
    const int nc = min(256, N - (int)blockIdx.x * 256);
    det_store(part, blockIdx.x, blockIdx.y, gridDim.y, 256, nc, sum8);
}

// ------------------------------------------------------------------------------------------------ embedding
// x[t,:] = drop(E[ids[t],:] * scale (+ pos[t % L,:]))  -> fp32 ; pad[t] = ids[t]==0   (hstu.py:124-128 ; sasrec.py:100-111)
// JAGGED (a packed SASRec batch): the position row of token t is tokpos[t] (sas_positions_kernel) instead of t % L, and a row
// outside every sequence (tokpos[t] < 0) gets x = 0 and pad = 1 whatever its id.
struct EmbedArgs {
    const long long* ids; const float* E; const float* pos;  // pos nullable [>=L, D]
    float* x; uint8_t* pad;
    int T, L, D; float scale; int mask_pad_rows;  // sasrec: x *= (id != 0)
    Dropout drop;
    const int* tokpos;   // JAGGED: [T] position row of each token, -1 = idle
};
template <bool JAGGED = false>
__global__ void __launch_bounds__(ROW_THREADS) embed_fwd_kernel(EmbedArgs a) {
    pdl_wait();
    a.drop.resolve();
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nw = gridDim.x * (ROW_THREADS / 32);
    for (int row = blockIdx.x * (ROW_THREADS / 32) + wib; row < a.T; row += nw) {
        long long id = a.ids[row];
        if constexpr (JAGGED) {
            if (a.tokpos[row] < 0) {
                if (lane == 0 && a.pad) a.pad[row] = 1;
                for (int c = lane * 4; c < a.D; c += 128) *reinterpret_cast<float4*>(a.x + (size_t)row * a.D + c) = make_float4(0.f, 0.f, 0.f, 0.f);
                continue;
            }
        }
        if (lane == 0 && a.pad) a.pad[row] = id == 0;
        const float* src = a.E + (size_t)id * a.D;
        const float* ps = a.pos ? a.pos + (size_t)(JAGGED ? a.tokpos[row] : row % a.L) * a.D : nullptr;
        const float keep = (a.mask_pad_rows && id == 0) ? 0.f : 1.f;
        for (int c = lane * 4; c < a.D; c += 128) {
            float4 v = *reinterpret_cast<const float4*>(src + c);
            float e[4] = {v.x * a.scale, v.y * a.scale, v.z * a.scale, v.w * a.scale};
            if (ps) {
                float4 p = *reinterpret_cast<const float4*>(ps + c);
                e[0] += p.x; e[1] += p.y; e[2] += p.z; e[3] += p.w;
            }
            size_t o = (size_t)row * a.D + c;
#pragma unroll
            for (int k = 0; k < 4; k += 2) {
                a.drop.apply2(e[k], e[k + 1], row, c + k);
                e[k] *= keep;
                e[k + 1] *= keep;
            }
            *reinterpret_cast<float4*>(a.x + o) = make_float4(e[0], e[1], e[2], e[3]);
        }
    }
}
// The longest sequence P of a packed batch, each sequence clamped to [0, T) and to L (seq_span), over one CTA's threads.
GRB_DEVINL int jagged_longest(const long long* offsets, int B, int T, int L, int* red) {
    int m = 0;
    for (int b = threadIdx.x; b < B; b += blockDim.x) {
        long long tok0;
        int len;
        seq_span(offsets, T, L, b, tok0, len);
        m = max(m, len);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    int P = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) P = max(P, red[w]);
    __syncthreads();
    return P;
}
// SASRec's position rule on a packed batch (one CTA): sasrec_collate_fn left-pads every sequence to P = the longest of the batch,
// so item i of a sequence of packed length n sits at position P - n + i.  tokpos[t] = that position for each sequence row and -1
// for every other row.  Every value is -1 or in [0, L), whatever the device offsets hold (overlapping sequences: one wins).
__global__ void __launch_bounds__(1024) sas_positions_kernel(const long long* __restrict__ offsets, int B, int T, int L,
                                                            int* __restrict__ tokpos) {
    pdl_wait();
    __shared__ int red[32];
    const int P = jagged_longest(offsets, B, T, L, red);
    for (int t = threadIdx.x; t < T; t += blockDim.x) tokpos[t] = -1;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    for (int b = threadIdx.x >> 5; b < B; b += blockDim.x >> 5) {
        long long tok0;
        int len;
        seq_span(offsets, T, L, b, tok0, len);
        for (int i = lane; i < len; i += 32) tokpos[tok0 + i] = P - len + i;
    }
}
struct EmbedBwdArgs {
    const long long* ids; const float* dx; float* dE; float* dpos;
    int T, L, D; float scale; int mask_pad_rows;
    Dropout drop;
    const long long* order;   // token indices sorted by id (stable)
};
// dpos[l,:] += sum over b = 0 .. B-1, in ascending b, of dropmask(dx[b L + l,:]) in fp32 (with mask_pad_rows, the tokens with id 0
// are left out), then one add of that sum per element: one CTA owns position row l and thread q its float4 column q, so the
// result does not depend on timing.  The CTA stages EMB_POS_STAGE float4 of the row's tokens at a time in shared memory (all of
// a chunk's loads in flight at once, 8 per thread), and the column owners add them in b order.
constexpr int EMB_POS_STAGE = 8 * ROW_THREADS;
__global__ void __launch_bounds__(ROW_THREADS) embed_bwd_pos_kernel(EmbedBwdArgs a) {
    __shared__ float4 stage[EMB_POS_STAGE];
    __shared__ uint8_t live[EMB_POS_STAGE];
    pdl_wait();
    a.drop.resolve();
    const int nq = a.D / 4, B = a.T / a.L, chunk = EMB_POS_STAGE / nq;   // D <= 256: chunk >= 32 tokens
    const int q = threadIdx.x;
    for (int l = blockIdx.x; l < a.L; l += gridDim.x) {
        float4* d = reinterpret_cast<float4*>(a.dpos + (size_t)l * a.D + 4 * q);
        const float4 o = q < nq ? *d : make_float4(0.f, 0.f, 0.f, 0.f);   // requested before the row's loads, added after its sum
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int b0 = 0; b0 < B; b0 += chunk) {
            const int nb = min(chunk, B - b0);
            float4 v[EMB_POS_STAGE / ROW_THREADS];
            bool pad[EMB_POS_STAGE / ROW_THREADS];
#pragma unroll
            for (int i = 0; i < EMB_POS_STAGE / ROW_THREADS; ++i) {
                const int e = threadIdx.x + i * ROW_THREADS, u = e / nq, c = 4 * (e - u * nq);
                const size_t row = (size_t)(b0 + u) * a.L + l;
                if (u < nb) v[i] = *reinterpret_cast<const float4*>(a.dx + row * a.D + c);
                pad[i] = u < nb && c == 0 && a.mask_pad_rows && a.ids[row] == 0;
            }
#pragma unroll
            for (int i = 0; i < EMB_POS_STAGE / ROW_THREADS; ++i) {
                const int e = threadIdx.x + i * ROW_THREADS, u = e / nq, c = 4 * (e - u * nq);
                if (u >= nb) continue;
                const int row = (b0 + u) * a.L + l;
                a.drop.apply2(v[i].x, v[i].y, row, c);
                a.drop.apply2(v[i].z, v[i].w, row, c + 2);
                stage[e] = v[i];
                if (c == 0) live[u] = !pad[i];
            }
            __syncthreads();
            if (q < nq) {
#pragma unroll 8
                for (int u = 0; u < nb; ++u) {
                    if (!live[u]) continue;
                    const float4 t = stage[u * nq + q];
                    s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
                }
            }
            __syncthreads();
        }
        if (q < nq) *d = make_float4(o.x + s.x, o.y + s.y, o.z + s.z, o.w + s.w);
    }
}

// embed_bwd_pos_kernel on a packed batch (a.T token rows, a.L = max_len): position row l < P (the longest sequence, jagged_longest)
// sums, in ascending b, dropmask(dx) of the token at position l of every sequence that reaches it (n_b >= P - l: row
// tok0_b + n_b - (P - l)), leaving out id-0 tokens with mask_pad_rows, then adds that sum once per element.  These are the
// terms, in the order, that embed_bwd_pos_kernel sums on the left-padded batch of the same sequences (whose other tokens at
// position l are pads), so the two give the same bits.  Rows l >= P are not written.
__global__ void __launch_bounds__(ROW_THREADS) embed_bwd_pos_jagged_kernel(EmbedBwdArgs a, const long long* __restrict__ offsets, int B) {
    __shared__ float4 stage[EMB_POS_STAGE];
    __shared__ uint8_t live[EMB_POS_STAGE];
    __shared__ int srow[EMB_POS_STAGE];
    __shared__ int red[ROW_THREADS / 32];
    pdl_wait();
    a.drop.resolve();
    const int nq = a.D / 4, chunk = EMB_POS_STAGE / nq;
    const int q = threadIdx.x;
    const int P = jagged_longest(offsets, B, a.T, a.L, red);
    for (int l = blockIdx.x; l < P; l += gridDim.x) {
        float4* d = reinterpret_cast<float4*>(a.dpos + (size_t)l * a.D + 4 * q);
        const float4 o = q < nq ? *d : make_float4(0.f, 0.f, 0.f, 0.f);
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int b0 = 0; b0 < B; b0 += chunk) {
            const int nb = min(chunk, B - b0);
            for (int u = threadIdx.x; u < nb; u += ROW_THREADS) {   // the token of sequence b0 + u at position l, or -1
                long long tok0;
                int len;
                seq_span(offsets, a.T, a.L, b0 + u, tok0, len);
                srow[u] = len >= P - l ? (int)(tok0 + len - (P - l)) : -1;
            }
            __syncthreads();
            float4 v[EMB_POS_STAGE / ROW_THREADS];
            bool pad[EMB_POS_STAGE / ROW_THREADS];
#pragma unroll
            for (int i = 0; i < EMB_POS_STAGE / ROW_THREADS; ++i) {
                const int e = threadIdx.x + i * ROW_THREADS, u = e / nq, c = 4 * (e - u * nq);
                const int row = u < nb ? srow[u] : -1;
                if (row >= 0) v[i] = *reinterpret_cast<const float4*>(a.dx + (size_t)row * a.D + c);
                pad[i] = u < nb && c == 0 && (row < 0 || (a.mask_pad_rows && a.ids[row] == 0));
            }
#pragma unroll
            for (int i = 0; i < EMB_POS_STAGE / ROW_THREADS; ++i) {
                const int e = threadIdx.x + i * ROW_THREADS, u = e / nq, c = 4 * (e - u * nq);
                if (u >= nb) continue;
                const int row = srow[u];
                if (row >= 0) {
                    a.drop.apply2(v[i].x, v[i].y, row, c);
                    a.drop.apply2(v[i].z, v[i].w, row, c + 2);
                    stage[e] = v[i];
                }
                if (c == 0) live[u] = !pad[i];
            }
            __syncthreads();
            if (q < nq) {
#pragma unroll 8
                for (int u = 0; u < nb; ++u) {
                    if (!live[u]) continue;
                    const float4 t = stage[u * nq + q];
                    s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
                }
            }
            __syncthreads();
        }
        if (q < nq) *d = make_float4(o.x + s.x, o.y + s.y, o.z + s.z, o.w + s.w);
    }
}

// dE[id,:] += sum over the tokens t with ids[t] == id, in token order, of scale * dropmask(dx[t,:]), with a summation order that does
// not depend on timing.  a.order lists the tokens sorted by id (stable) and is cut into fixed pieces of 32 positions:
//   pass 1 (one warp per piece): the tokens of every id run inside the piece are summed in order -> piece[first position][:]
//   pass 2 (one warp per id run): the run's pieces are summed in order and added to dE once
struct EmbedPieceArgs {
    EmbedBwdArgs e;
    float* piece;   // [T, D] fp32 scratch, rows indexed by sorted position
};
// (the warp-wide shuffles / ballots sit outside the column loops: with D = 64 half of the lanes own no column)
constexpr int EMB_MAX_CH = 2;   // float4 columns per lane: D <= 256
__global__ void __launch_bounds__(ROW_THREADS) embed_bwd_piece_kernel(EmbedPieceArgs a) {
    pdl_wait();
    a.e.drop.resolve();
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nw = gridDim.x * (ROW_THREADS / 32);
    const int npieces = (a.e.T + 31) / 32;
    for (int k = blockIdx.x * (ROW_THREADS / 32) + wib; k < npieces; k += nw) {
        const int q = k * 32 + lane;
        const int rowq = q < a.e.T ? (int)a.e.order[q] : 0;
        const long long idq = q < a.e.T ? a.e.ids[rowq] : -1;
        const int cnt = min(32, a.e.T - k * 32);
        float4 s[EMB_MAX_CH];
#pragma unroll
        for (int h = 0; h < EMB_MAX_CH; ++h) s[h] = make_float4(0.f, 0.f, 0.f, 0.f);
        int start = 0;
        for (int j = 0; j < cnt; ++j) {
            const int row = __shfl_sync(0xffffffffu, rowq, j);
            const long long id = __shfl_sync(0xffffffffu, idq, j);
            const long long next = __shfl_sync(0xffffffffu, idq, (j + 1) & 31);
            const bool last = j + 1 == cnt || next != id;
#pragma unroll
            for (int h = 0; h < EMB_MAX_CH; ++h) {
                const int c = 4 * lane + 128 * h;
                if (c >= a.e.D) continue;
                float4 v = *reinterpret_cast<const float4*>(a.e.dx + (size_t)row * a.e.D + c);
                a.e.drop.apply2(v.x, v.y, row, c);
                a.e.drop.apply2(v.z, v.w, row, c + 2);
                s[h].x += v.x * a.e.scale; s[h].y += v.y * a.e.scale; s[h].z += v.z * a.e.scale; s[h].w += v.w * a.e.scale;
                if (last) {
                    *reinterpret_cast<float4*>(a.piece + (size_t)(k * 32 + start) * a.e.D + c) = s[h];
                    s[h] = make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
            if (last) start = j + 1;
        }
    }
}
__global__ void __launch_bounds__(ROW_THREADS) embed_bwd_run_kernel(EmbedPieceArgs a) {
    pdl_wait();
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int nw = gridDim.x * (ROW_THREADS / 32);
    const int T = a.e.T;
    for (int p = blockIdx.x * (ROW_THREADS / 32) + wib; p < T; p += nw) {
        const long long id = a.e.ids[a.e.order[p]];
        if (id == 0 || (p > 0 && a.e.ids[a.e.order[p - 1]] == id)) continue;
        float4 s[EMB_MAX_CH];
#pragma unroll
        for (int h = 0; h < EMB_MAX_CH; ++h) {
            const int c = 4 * lane + 128 * h;
            s[h] = c < a.e.D ? *reinterpret_cast<const float4*>(a.piece + (size_t)p * a.e.D + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        // the further pieces of the run start at the piece boundaries 32 k > p whose first token still has this id
        for (int k0 = p / 32 + 1; k0 * 32 < T; k0 += 32) {
            const int k = k0 + lane;
            const bool match = k * 32 < T && a.e.ids[a.e.order[k * 32]] == id;
            const unsigned miss = ~__ballot_sync(0xffffffffu, match);
            const int cnt = miss ? __ffs(miss) - 1 : 32;
            for (int j = 0; j < cnt; ++j) {
#pragma unroll
                for (int h = 0; h < EMB_MAX_CH; ++h) {
                    const int c = 4 * lane + 128 * h;
                    if (c >= a.e.D) continue;
                    const float4 v = *reinterpret_cast<const float4*>(a.piece + (size_t)(k0 + j) * 32 * a.e.D + c);
                    s[h].x += v.x; s[h].y += v.y; s[h].z += v.z; s[h].w += v.w;
                }
            }
            if (cnt < 32) break;
        }
#pragma unroll
        for (int h = 0; h < EMB_MAX_CH; ++h) {
            const int c = 4 * lane + 128 * h;
            if (c < a.e.D) red_add_v4(a.e.dE + (size_t)id * a.e.D + c, s[h].x, s[h].y, s[h].z, s[h].w);
        }
    }
}

// ------------------------------------------------------------------------------------------------ cross entropy on bf16 logits
// count = #(targets != 0)  -> inv_count (0 if none); loss <- 0, or NaN when no target is valid (F.cross_entropy's 0 / 0 mean,
// hstu.py:141-146; the gradients of such a batch are zero here, NaN in the reference)
__global__ void ce_count_kernel(const long long* __restrict__ tg, int T, float* __restrict__ inv_count, float* __restrict__ loss) {
    pdl_wait();
    __shared__ int red[32];
    int c = 0;
    // 16-byte loads, deeply unrolled: all loads of a thread are in flight together (this single-CTA kernel is one DRAM
    // round trip long instead of one per target)
    const longlong2* tg2 = reinterpret_cast<const longlong2*>(tg);
    const int T2 = ((reinterpret_cast<uintptr_t>(tg) & 15) == 0) ? T / 2 : 0;
#pragma unroll 16
    for (int i = threadIdx.x; i < T2; i += blockDim.x) {
        const longlong2 v = tg2[i];
        c += (v.x != 0) + (v.y != 0);
    }
    for (int i = 2 * T2 + threadIdx.x; i < T; i += blockDim.x) c += tg[i] != 0;
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int s = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += red[w];
        *inv_count = s > 0 ? 1.f / (float)s : 0.f;
        *loss = s > 0 ? 0.f : __int_as_float(0x7fc00000);
    }
}
// one CTA per row: loss += (lse - logit[target]) * inv_count ; logits <- (softmax - onehot) * inv_count  (0 for ignored rows)
// pad columns [C, ld) are written with zeros.   (hstu.py:141-146, ignore_index = 0, class 0 stays in the denominator)
// src32 (nullable, [T, ld] fp32): the logits are read from there instead of `logits`, which then only receives the gradient -
// fp32 logits keep the softmax exact when a row spans tens of nats (bf16 rounds a logit of 60 by 0.25).
__global__ void __launch_bounds__(256) ce_fwd_bwd_kernel(bf16* __restrict__ logits, int ld, int C, const long long* __restrict__ tg,
                                                        const float* __restrict__ inv_count, float* __restrict__ row_loss,
                                                        int write_grad, const float* __restrict__ src32) {
    pdl_wait();
    __shared__ float red[8];
    __shared__ float bc[2];
    const int row = blockIdx.x, tid = threadIdx.x;
    bf16* lr = logits + (size_t)row * ld;
    const float* sr = src32 ? src32 + (size_t)row * ld : nullptr;
    auto logit = [&](int c) { return sr ? sr[c] : __bfloat162float(lr[c]); };
    const long long t = tg[row];
    const float ic = *inv_count;
    if (t == 0) {
        if (tid == 0) row_loss[row] = 0.f;
        if (write_grad)
            for (int c = tid; c < ld; c += 256) lr[c] = __float2bfloat16(0.f);
        return;
    }
    float m = -INFINITY;
    for (int c = tid; c < C; c += 256) m = fmaxf(m, logit(c));
    m = warp_max(m);
    if ((tid & 31) == 0) red[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) {
        float mm = red[0];
        for (int w = 1; w < 8; ++w) mm = fmaxf(mm, red[w]);
        bc[0] = mm;
    }
    __syncthreads();
    m = bc[0];
    float s = 0.f;
    for (int c = tid; c < C; c += 256) s += __expf(logit(c) - m);
    s = warp_sum(s);
    __syncthreads();
    if ((tid & 31) == 0) red[tid >> 5] = s;
    __syncthreads();
    if (tid == 0) {
        float ss = 0.f;
        for (int w = 0; w < 8; ++w) ss += red[w];
        bc[1] = ss;
        float lse = m + logf(ss);
        row_loss[row] = (lse - logit((int)t)) * ic;
    }
    __syncthreads();
    if (!write_grad) return;
    const float inv_s = 1.f / bc[1];
    for (int c = tid; c < ld; c += 256) {
        float gvl = 0.f;
        if (c < C) {
            gvl = __expf(logit(c) - m) * inv_s;
            if (c == (int)t) gvl -= 1.f;
            gvl *= ic;
        }
        lr[c] = __float2bfloat16(gvl);
    }
}

// loss += sum of the per-row losses, in a fixed order (one CTA of 1024 threads: strided partial sums, then a fixed tree)
__global__ void __launch_bounds__(1024) ce_loss_sum_kernel(const float* __restrict__ row_loss, int T, float* __restrict__ loss) {
    pdl_wait();
    __shared__ float red[32];
    float s = 0.f;
    for (int i = threadIdx.x; i < T; i += 1024) s += row_loss[i];
    s = warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x < 32) {
        s = warp_sum(red[threadIdx.x]);
        if (threadIdx.x == 0) *loss += s;
    }
}

// Register-resident variant: the whole row (<= 256 x NCH x 8 logits) is read ONCE with 16-byte loads; exp(x - max) is
// evaluated once per logit and kept in registers for the gradient pass; the row is written ONCE.
// HBM traffic = 1 read + 1 write of the logits; ~10 instructions per logit.  src32: as in ce_fwd_bwd_kernel.
template <int NCH>
__global__ void __launch_bounds__(256) ce_fwd_bwd_vec_kernel(bf16* __restrict__ logits, int ld, int C, const long long* __restrict__ tg,
                                                            const float* __restrict__ inv_count, float* __restrict__ row_loss, int write_grad,
                                                            const float* __restrict__ src32) {
    pdl_wait();
    __shared__ float red[8];
    __shared__ float bc[3];
    const int row = blockIdx.x, tid = threadIdx.x;
    uint4* lr = reinterpret_cast<uint4*>(logits + (size_t)row * ld);
    const int nchunks = ld >> 3;
    const int t = (int)tg[row];
    const float ic = *inv_count;
    if (t == 0) {
        if (tid == 0) row_loss[row] = 0.f;
        if (write_grad)
            for (int c = tid; c < nchunks; c += 256) lr[c] = make_uint4(0u, 0u, 0u, 0u);
        return;
    }
    float e[NCH][8];
    float m = -INFINITY;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
        const int c = tid + i * 256;
        if (c < nchunks) {
            if (src32) {
                const float4* sr = reinterpret_cast<const float4*>(src32 + (size_t)row * ld) + 2 * c;
                const float4 f0 = sr[0], f1 = sr[1];
                e[i][0] = f0.x; e[i][1] = f0.y; e[i][2] = f0.z; e[i][3] = f0.w;
                e[i][4] = f1.x; e[i][5] = f1.y; e[i][6] = f1.z; e[i][7] = f1.w;
            } else {
                const uint4 q = lr[c];
                const uint32_t u[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    float2 f = unpack_bf16(u[k]);
                    e[i][2 * k] = f.x;
                    e[i][2 * k + 1] = f.y;
                }
            }
            if (c * 8 + 8 > C) {   // the single partial chunk: pad columns do not take part
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    if (c * 8 + k >= C) e[i][k] = -INFINITY;
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) m = fmaxf(m, e[i][k]);
        }
    }
    m = warp_max(m);
    if ((tid & 31) == 0) red[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) {
        float mm = red[0];
        for (int w = 1; w < 8; ++w) mm = fmaxf(mm, red[w]);
        bc[0] = mm;
    }
    __syncthreads();
    m = bc[0];
    const float ml2 = m * 1.4426950408889634f;
    float ssum = 0.f;
    // the thread that owns the target column remembers its logit
    const int tc = t >> 3, ti = (tc - tid) >> 8;
    float tlogit = 0.f;
    const bool own = (tc >= tid) && (((tc - tid) & 255) == 0) && ti < NCH;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
        const int c = tid + i * 256;
        if (c < nchunks) {
            if (own && i == ti) {
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    if (k == (t & 7)) tlogit = e[i][k];
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                e[i][k] = exp2f(fmaf(e[i][k], 1.4426950408889634f, -ml2));   // exp(x - m); exp2(-inf) = 0 for pad columns
                ssum += e[i][k];
            }
        }
    }
    ssum = warp_sum(ssum);
    __syncthreads();
    if ((tid & 31) == 0) red[tid >> 5] = ssum;
    __syncthreads();
    if (tid == 0) {
        float ss = 0.f;
        for (int w = 0; w < 8; ++w) ss += red[w];
        bc[1] = ss;
    }
    __syncthreads();
    const float stot = bc[1];
    if (own) row_loss[row] = (m + logf(stot) - tlogit) * ic;
    if (!write_grad) return;
    const float sc = ic / stot;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
        const int c = tid + i * 256;
        if (c < nchunks) {
            float gk[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) gk[k] = e[i][k] * sc;
            if (own && i == ti) {
#pragma unroll
                for (int k = 0; k < 8; ++k)
                    if (k == (t & 7)) gk[k] -= ic;
            }
            lr[c] = make_uint4(pack_bf16(gk[0], gk[1]), pack_bf16(gk[2], gk[3]), pack_bf16(gk[4], gk[5]), pack_bf16(gk[6], gk[7]));
        }
    }
}

// ------------------------------------------------------------------------------------------------ fused Adam (torch.optim.Adam semantics)
// state[0] = step (as float), state[1] = 1 - beta1^step, state[2] = 1 - beta2^step ; ticked on device so a CUDA graph replays correctly
__global__ void adam_tick_kernel(float* state, float beta1, float beta2) {
    pdl_wait();
    float step = state[0] + 1.f;
    state[0] = step;
    state[1] = 1.f - powf(beta1, step);
    state[2] = 1.f - powf(beta2, step);
}
struct AdamArgs {
    float* p; float* g; float* m; float* v; bf16* p_bf16;  // p_bf16 nullable
    size_t n;
    const float* state;
    float lr, beta1, beta2, eps, weight_decay, grad_scale;
    int zero_grad;
};
// One element of the step: p, and m / v in place, from the raw gradient g.  adam_step_kernel and the lazy table step
// (lazy_adam.cuh) both call it, so an element gets the same bits from either.
GRB_DEVINL float adam_update(float p, float g, float& m, float& v, float grad_scale, float beta1, float beta2, float eps,
                             float weight_decay, float step_size, float inv_sqrt_bc2) {
    g *= grad_scale;
    if (weight_decay != 0.f) g += weight_decay * p;
    m = beta1 * m + (1.f - beta1) * g;
    v = beta2 * v + (1.f - beta2) * g * g;
    float denom = sqrtf(v) * inv_sqrt_bc2 + eps;
    return p - step_size * (m / denom);
}
__global__ void adam_step_kernel(AdamArgs a) {
    pdl_wait();
    const float bc1 = a.state[1], bc2 = a.state[2];
    const float step_size = a.lr / bc1;
    const float inv_sqrt_bc2 = rsqrtf(bc2);
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < a.n; i += stride) {
        float m = a.m[i], v = a.v[i];
        const float p = adam_update(a.p[i], a.g[i], m, v, a.grad_scale, a.beta1, a.beta2, a.eps, a.weight_decay, step_size, inv_sqrt_bc2);
        a.m[i] = m;
        a.v[i] = v;
        a.p[i] = p;
        if (a.p_bf16) a.p_bf16[i] = __float2bfloat16(p);
        if (a.zero_grad) a.g[i] = 0.f;
    }
}
__global__ void cast_flat_f32_bf16_kernel(const float* __restrict__ in, bf16* __restrict__ out, size_t n) {
    pdl_wait();
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    size_t stride = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += stride) out[i] = __float2bfloat16(in[i]);
}


// ------------------------------------------------------------------------------------------------ split-bf16 operands
// fp32-accurate GEMM on the bf16 tensor path: x = hi + mid + lo with three bf16 terms (24 mantissa bits together); the product
// of two such numbers keeps the six terms of weight >= 2^-16 (hi*hi, hi*mid, mid*hi, hi*lo, lo*hi, mid*mid).  Laying the terms
// out along K,   A' = [hi | hi | mid | hi | lo | mid]   B' = [hi | mid | hi | lo | hi | mid]   (K' = 6 K),
// turns the sum of the six partial GEMMs into ONE ordinary GEMM with fp32 accumulation.
// out [rows, 6 K] bf16 ; operand 0 = A layout, 1 = B layout.
__global__ void __launch_bounds__(256) split3_f32_bf16_kernel(const float* __restrict__ in, bf16* __restrict__ out, size_t rows, int K, int operand) {
    pdl_wait();
    const size_t n = rows * (size_t)K;
    for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
        const size_t r = e / K;
        const int k = (int)(e % K);
        const float x = in[e];
        const bf16 hi = __float2bfloat16_rn(x);
        const float r1 = x - __bfloat162float(hi);
        const bf16 mid = __float2bfloat16_rn(r1);
        const bf16 lo = __float2bfloat16_rn(r1 - __bfloat162float(mid));
        bf16* o = out + r * (size_t)(6 * K) + k;
        if (operand == 0) { o[0] = hi; o[K] = hi; o[2 * K] = mid; o[3 * K] = hi; o[4 * K] = lo; o[5 * K] = mid; }
        else              { o[0] = hi; o[K] = mid; o[2 * K] = hi; o[3 * K] = lo; o[4 * K] = hi; o[5 * K] = mid; }
    }
}


// ------------------------------------------------------------------------------------------------ leave-one-out metrics
// Replaces the per-sample Python loop of genrec/trainers/hstu_trainer.py:55-81 (`logits[:, 0] = -inf`, top-k, `.item()` per
// sample): the rank of the held-out target among classes 1..C-1 is counted directly - rank = 1 + #{j >= 1 : logit_j > logit_t or
// (logit_j == logit_t and j < t)} (torch.topk's order on ties: lower index first) - and Recall@k / NDCG@k for k in {1, 5, 10}
// are ACCUMULATED on the device:  out[0..2] += hit@{1,5,10}, out[3..5] += ndcg@{1,5,10}.  One CTA per sample; targets of 0
// (padding) contribute nothing.  ranks (nullable) receives the per-sample rank (0 for skipped samples).
// One ranked sample's share of the sums; the fused head (head_rank.cuh) adds its samples with the same expressions.
GRB_DEVINL void rank_metrics_add(float* out, int rank) {
    const float nd = 1.f / log2f((float)rank + 1.f);
    if (rank <= 1) { atomicAdd(out + 0, 1.f); atomicAdd(out + 3, nd); }
    if (rank <= 5) { atomicAdd(out + 1, 1.f); atomicAdd(out + 4, nd); }
    if (rank <= 10) { atomicAdd(out + 2, 1.f); atomicAdd(out + 5, nd); }
}
__global__ void __launch_bounds__(256) eval_rank_kernel(const float* __restrict__ logits, int C, const long long* __restrict__ targets,
                                                       float* __restrict__ out, int* __restrict__ ranks) {
    pdl_wait();
    __shared__ int red[8];
    const int b = blockIdx.x;
    const long long t = targets[b];
    if (t <= 0 || t >= C) {
        if (threadIdx.x == 0 && ranks) ranks[b] = 0;
        return;
    }
    const float* row = logits + (size_t)b * C;
    const float lt = row[t];
    int c = 0;
    for (int j = 1 + threadIdx.x; j < C; j += 256) {
        const float v = row[j];
        c += (v > lt) || (v == lt && j < (int)t);
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int rank = 1;
        for (int w = 0; w < 8; ++w) rank += red[w];
        if (ranks) ranks[b] = rank;
        rank_metrics_add(out, rank);
    }
}


// ------------------------------------------------------------------------------------------------ jagged -> left-padded batch
// Device-side hstu_collate_fn (genrec/data/amazon_hstu.py:137-173): user b's history is items[offsets[b] .. offsets[b+1]) (time
// order) with the held-out target targets[b].  With n = min(len_b, L) kept (the LAST n events) and pad = L - n:
//   input_ids[b, p]  = p < pad ? 0 : hist[p - pad]          timestamps[b, p] = p < pad ? 0 : ts[p - pad]
//   targets[b, p]    = p + 1 < pad ? 0 : (p + 1 - pad < n ? hist[p + 1 - pad] : target_b)      (the sequence shifted by one)
// One thread per output position; stamps / out_ts may be null (SASRec: genrec/data/amazon_sasrec.py:125-161).
__global__ void __launch_bounds__(256) collate_jagged_kernel(const long long* __restrict__ items, const long long* __restrict__ stamps,
                                                            const long long* __restrict__ offsets, const long long* __restrict__ targets, int B,
                                                            int L, long long* __restrict__ out_ids, long long* __restrict__ out_tg,
                                                            long long* __restrict__ out_ts) {
    pdl_wait();
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= (size_t)B * L) return;
    const int b = (int)(e / L), p = (int)(e % L);
    const long long lo = offsets[b], hi = offsets[b + 1];
    const long long len = hi - lo;
    const int n = (int)(len < L ? len : L);
    const int pad = L - n;
    const long long* h = items + (hi - n);            // the last n events
    out_ids[e] = p < pad ? 0 : h[p - pad];
    out_tg[e] = p + 1 < pad ? 0 : (p + 1 - pad < n ? h[p + 1 - pad] : targets[b]);
    if (out_ts != nullptr) out_ts[e] = (p < pad || stamps == nullptr) ? 0 : stamps[(hi - n) + (p - pad)];
}

// ------------------------------------------------------------------------------------------------ jagged -> packed batch
// The rows of collate_jagged_kernel without their pads: sequence b keeps n_b = min(len_b, max_seq_len) rows (its LAST n_b events),
// packed one after another from row 0.  out_off [B+1] = the running sum of n_b, clamped to T; info[0] = the unclamped total (> T:
// the batch did not fit and its tail was cut), info[1] = the longest n_b.  One CTA.
__global__ void __launch_bounds__(1024) pack_jagged_offsets_kernel(const long long* __restrict__ offsets, int B, int max_seq_len, int T,
                                                                  long long* __restrict__ out_off, long long* __restrict__ info) {
    pdl_wait();
    __shared__ long long warp_sum[32];
    __shared__ long long s_carry;
    __shared__ int warp_max[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) { s_carry = 0; out_off[0] = 0; }
    int mx = 0;
    for (int base = 0; base < B; base += 1024) {
        __syncthreads();                                   // s_carry of the previous chunk is visible, warp_sum free
        const long long carry = s_carry;
        const int b = base + threadIdx.x;
        long long n = 0;
        if (b < B) {
            n = offsets[b + 1] - offsets[b];
            n = n < 0 ? 0 : (n > max_seq_len ? max_seq_len : n);
        }
        mx = max(mx, (int)n);
        long long v = n;                                   // inclusive scan: lanes, then warps
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long u = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += u;
        }
        if (lane == 31) warp_sum[warp] = v;
        __syncthreads();
        long long before = 0;
        for (int w = 0; w < warp; ++w) before += warp_sum[w];
        const long long incl = carry + before + v;
        if (b < B) out_off[b + 1] = incl < T ? incl : T;
        __syncthreads();                                   // every thread has read s_carry and warp_sum
        if (threadIdx.x == 1023) s_carry = incl;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) warp_max[warp] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
        int m = 0;
        for (int w = 0; w < 32; ++w) m = max(m, warp_max[w]);
        info[0] = s_carry;
        info[1] = m;
    }
}
// Row t < out_off[B] of sequence b (out_off[b] <= t < out_off[b+1]), p = t - out_off[b], n = its packed length:
//   input_ids[t] = hist[p]    timestamps[t] = ts[p]    targets[t] = p + 1 < n ? hist[p + 1] : target_b
// with hist / ts the last n events of user b; rows t >= out_off[B] are idle (id 0, target 0, timestamp 0).
__global__ void __launch_bounds__(256) pack_jagged_kernel(const long long* __restrict__ items, const long long* __restrict__ stamps,
                                                         const long long* __restrict__ offsets, const long long* __restrict__ targets,
                                                         const long long* __restrict__ out_off, int B, int T, long long* __restrict__ out_ids,
                                                         long long* __restrict__ out_tg, long long* __restrict__ out_ts) {
    pdl_wait();
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    long long id = 0, tg = 0, ts = 0;
    if (t < out_off[B]) {
        int lo = 0, hi = B - 1;                            // the first b with out_off[b + 1] > t
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (out_off[mid + 1] > t) hi = mid; else lo = mid + 1;
        }
        const long long p = t - out_off[lo], n = out_off[lo + 1] - out_off[lo];
        const long long src = offsets[lo + 1] - n + p;
        id = items[src];
        tg = p + 1 < n ? items[src + 1] : targets[lo];
        ts = stamps != nullptr ? stamps[src] : 0;
    }
    out_ids[t] = id;
    out_tg[t] = tg;
    if (out_ts != nullptr) out_ts[t] = ts;
}


}  // namespace grb
