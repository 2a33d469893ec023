// genrec_b200 - fp32-exact forward path of the HSTU block (north_star: "1e-5 (fp32)").
//
// The bf16 kernels follow what the reference does under Accelerator(mixed_precision="bf16"); this path follows what it does WITHOUT
// autocast (plain fp32 modules, genrec/models/hstu.py:222-280): every linear layer is the split-bf16 tensor-core GEMM of api.cu
// (three bf16 terms per operand, six cross products, fp32 accumulation: fp32-accurate), everything between the GEMMs is fp32:
//   hstu_attn_f32_fwd_kernel   O = silu(Q K^T + bias) V on the CUDA cores (exact products, fp32 accumulation)
//   ln_gate_f32_kernel         x1 = x + LN1(O) * U ; xn = LN2(x1)
//   ln_f32_kernel              final LayerNorm
// Forward only (inference / evaluation / parity): training keeps the bf16 path.
#pragma once
#include "attn_hstu.cuh"
#include "tc_gemm.cuh"

namespace grb {

GRB_DEVINL float silu_exact(float z) { return __fdiv_rn(z, 1.f + exp_accurate(-z)); }

struct HstuAttnF32Args {
    const float* P;   // [T, ld]  U | V | Q | K, each D wide, head h = columns h*DH .. (after SiLU)
    int ld;
    int B, L, H;
    HstuBiasArgs bias;   // [B, L, ldix] uint16 index matrix (built once per batch by hstu_bias_index_kernel)
    float* O;         // [T, D]
};

constexpr int AF_ROWS = 32, AF_KEYS = 64, AF_THREADS = 128;

// grid (ceil(L / 32), B * H).  Thread (r = tid / 4, kq = tid % 4): query row r of the tile, keys kq, kq + 4, ... of every key tile;
// the four partial output rows meet through shuffles.  q and the output partial live in registers, K / V tiles in shared memory.
template <int DH>
__global__ void __launch_bounds__(AF_THREADS) hstu_attn_f32_fwd_kernel(HstuAttnF32Args a) {
    pdl_wait();
    extern __shared__ float af_smem[];
    float* Ks = af_smem;                       // [64][DH]
    float* Vs = Ks + AF_KEYS * DH;             // [64][DH]
    float* wcomb = Vs + AF_KEYS * DH;          // [npos * 64 + 1]
    const int tid = threadIdx.x, r = tid >> 2, kq = tid & 3;
    const int b = blockIdx.y / a.H, h = blockIdx.y % a.H;
    const int D = a.H * DH;
    const int q0 = blockIdx.x * AF_ROWS, i = q0 + r;
    const unsigned sentinel = (unsigned)a.bias.npos * 64u;
    {
        const int n = a.bias.npos * 64;
        for (int e = tid; e < n; e += AF_THREADS) {
            const int pb = e >> 6, tb = e & 63;
            float v = a.bias.wpos[pb * a.H + h];
            if (a.bias.wtime && tb < a.bias.ntime) v += a.bias.wtime[tb * a.H + h];
            wcomb[e] = v;
        }
    }
    const size_t tok0 = (size_t)b * a.L;
    float q[DH], o[DH];
#pragma unroll
    for (int d = 0; d < DH; ++d) { q[d] = 0.f; o[d] = 0.f; }
    if (i < a.L) {
        const float4* src = reinterpret_cast<const float4*>(a.P + (tok0 + i) * a.ld + 2 * D + h * DH);
#pragma unroll
        for (int d4 = 0; d4 < DH / 4; ++d4) { const float4 t = src[d4]; q[4 * d4] = t.x; q[4 * d4 + 1] = t.y; q[4 * d4 + 2] = t.z; q[4 * d4 + 3] = t.w; }
    }
    const uint16_t* ix = a.bias.bias_index + (tok0 + (i < a.L ? i : 0)) * a.bias.ldix;
    const int kend = min(a.L, q0 + AF_ROWS);   // causal: no key beyond the last query row of this tile
    for (int j0 = 0; j0 < kend; j0 += AF_KEYS) {
        __syncthreads();
        for (int e = tid; e < AF_KEYS * (DH / 4); e += AF_THREADS) {
            const int jj = e / (DH / 4), d4 = e % (DH / 4);
            float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
            if (j0 + jj < a.L) {
                const float* row = a.P + (tok0 + j0 + jj) * a.ld + h * DH;
                kv = reinterpret_cast<const float4*>(row + 3 * D)[d4];
                vv = reinterpret_cast<const float4*>(row + D)[d4];
            }
            reinterpret_cast<float4*>(Ks + jj * DH)[d4] = kv;
            reinterpret_cast<float4*>(Vs + jj * DH)[d4] = vv;
        }
        __syncthreads();
        if (i < a.L) {
            const int jmax = min(AF_KEYS, i - j0 + 1);   // keys j <= i
            for (int jj = kq; jj < jmax; jj += 4) {
                const unsigned id = ix[j0 + jj];
                if (id == sentinel) continue;             // masked cell: silu(-1e9) is an exact zero in the reference (hstu.py:257-264)
                const float* kr = Ks + jj * DH;
                float s = 0.f;
#pragma unroll
                for (int d = 0; d < DH; ++d) s = fmaf(q[d], kr[d], s);
                const float w = silu_exact(s + wcomb[id]);
                const float* vr = Vs + jj * DH;
#pragma unroll
                for (int d = 0; d < DH; ++d) o[d] = fmaf(w, vr[d], o[d]);
            }
        }
    }
#pragma unroll
    for (int d = 0; d < DH; ++d) {
        o[d] += __shfl_xor_sync(0xffffffffu, o[d], 1);
        o[d] += __shfl_xor_sync(0xffffffffu, o[d], 2);
    }
    if (i < a.L) {
        float* dst = a.O + (tok0 + i) * D + h * DH;
#pragma unroll
        for (int d = 0; d < DH; ++d)
            if ((d & 3) == kq) dst[d] = o[d];   // static register indices; every thread of the quad stores a quarter
    }
}

template <int DH>
inline cudaError_t launch_hstu_attn_f32(const HstuAttnF32Args& a, cudaStream_t st) {
    const size_t smem = (size_t)(2 * AF_KEYS * DH + a.bias.npos * 64 + 1) * sizeof(float);
    dim3 grid((a.L + AF_ROWS - 1) / AF_ROWS, a.B * a.H);
    return launch_k(hstu_attn_f32_fwd_kernel<DH>, grid, AF_THREADS, smem, st, a);
}

// ------------------------------------------------------------------------------------------------ fp32 row kernels (one warp per row)
template <int NP>   // D = 32 * NP
GRB_DEVINL void ln_row_f32(const float (&v)[NP], const float* g, const float* b, int lane, float eps, float (&out)[NP]) {
    float s = 0.f;
#pragma unroll
    for (int p = 0; p < NP; ++p) s += v[p];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = __fdiv_rn(s, (float)(32 * NP));
    float q = 0.f;
#pragma unroll
    for (int p = 0; p < NP; ++p) { const float d = v[p] - mean; q = fmaf(d, d, q); }
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = __fdiv_rn(1.f, __fsqrt_rn(__fdiv_rn(q, (float)(32 * NP)) + eps));   // (the library is built with --use_fast_math)
#pragma unroll
    for (int p = 0; p < NP; ++p) out[p] = (v[p] - mean) * rstd * g[p * 32 + lane] + b[p * 32 + lane];
}
struct LnGateF32Args {
    const float* O; const float* U; int ldu; const float* x;
    const float* g1; const float* b1; const float* g2; const float* b2;
    float* x1; float* xn;   // xn nullable
    int T; float eps;
};
// x1 = x + LN1(O) * U ; xn = LN2(x1)      (hstu.py:271-278, eval mode: dropout is the identity)
template <int NP>
__global__ void __launch_bounds__(256) ln_gate_f32_kernel(LnGateF32Args a) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    constexpr int D = 32 * NP;
    for (int row = blockIdx.x * 8 + (threadIdx.x >> 5); row < a.T; row += gridDim.x * 8) {
        float v[NP], y[NP];
#pragma unroll
        for (int p = 0; p < NP; ++p) v[p] = a.O[(size_t)row * D + p * 32 + lane];
        ln_row_f32<NP>(v, a.g1, a.b1, lane, a.eps, y);
#pragma unroll
        for (int p = 0; p < NP; ++p) {
            y[p] = a.x[(size_t)row * D + p * 32 + lane] + y[p] * a.U[(size_t)row * a.ldu + p * 32 + lane];
            a.x1[(size_t)row * D + p * 32 + lane] = y[p];
        }
        if (a.xn) {
            ln_row_f32<NP>(y, a.g2, a.b2, lane, a.eps, v);
#pragma unroll
            for (int p = 0; p < NP; ++p) a.xn[(size_t)row * D + p * 32 + lane] = v[p];
        }
    }
}
template <int NP>
__global__ void __launch_bounds__(256) ln_f32_kernel(const float* __restrict__ x, const float* __restrict__ g, const float* __restrict__ b,
                                                     float* __restrict__ y, int T, float eps) {
    pdl_wait();
    const int lane = threadIdx.x & 31;
    constexpr int D = 32 * NP;
    for (int row = blockIdx.x * 8 + (threadIdx.x >> 5); row < T; row += gridDim.x * 8) {
        float v[NP], o[NP];
#pragma unroll
        for (int p = 0; p < NP; ++p) v[p] = x[(size_t)row * D + p * 32 + lane];
        ln_row_f32<NP>(v, g, b, lane, eps, o);
#pragma unroll
        for (int p = 0; p < NP; ++p) y[(size_t)row * D + p * 32 + lane] = o[p];
    }
}

}  // namespace grb
