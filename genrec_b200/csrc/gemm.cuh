// genrec_b200 - generic bf16 tensor-core GEMM with fused epilogues (first-generation path: cp.async + ldmatrix +
// mma.sync.m16n8k16; the wgmma/TMA kernels in tc_*.cuh replace it on the hot GEMMs).
//
//   C[M,N] (+)= opA(A) * opB(B),  fp32 accumulate
//     AMODE 0 : A stored [M][K], K contiguous          AMODE 1 : A stored [K][M], M contiguous (i.e. A^T given)
//     BMODE 0 : B stored [N][K], K contiguous (nn.Linear weight for x*W^T)
//     BMODE 1 : B stored [K][N], N contiguous
//   grid = (ceil(N/128), ceil(M/128), splitK).  Requirements: lda/ldb multiples of 8 elements, 16-byte aligned bases.
#pragma once
#include "common.cuh"

namespace grb {

constexpr int GEMM_BM = 128, GEMM_BN = 128, GEMM_BK = 32, GEMM_STAGES = 3, GEMM_THREADS = 256;
constexpr int GEMM_LDK = GEMM_BK + 8;    // padded row (elements) of a K-contiguous tile  [128][40]
constexpr int GEMM_LDMN = GEMM_BM + 8;   // padded row of an MN-contiguous tile             [32][136]
constexpr int GEMM_TILE_ELEMS = (GEMM_BM * GEMM_LDK > GEMM_BK * GEMM_LDMN) ? GEMM_BM * GEMM_LDK : GEMM_BK * GEMM_LDMN;
constexpr int GEMM_SMEM_BYTES = 2 * GEMM_STAGES * GEMM_TILE_ELEMS * 2;

struct GemmShape {
    int M, N, K;
    int lda, ldb;
    int k_per_split;  // multiple of GEMM_BK ; == roundup(K) when no split
};

// Loads one 128 x 32 (mn x k) operand tile into smem.  MODE 0: gmem [mn][k]; MODE 1: gmem [k][mn].
template <int MODE>
GRB_DEVINL void gemm_load_tile(bf16* __restrict__ s, const bf16* __restrict__ g, int ld, int mn0, int mn_max, int k0,
                               int k_max, int tid) {
    if (MODE == 0) {
        // 128 rows x 4 chunks(16B) = 512 chunks ; 256 threads x 2
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            int c = tid + i * GEMM_THREADS;
            int r = c >> 2, kc = (c & 3) * 8;
            int gr = mn0 + r, gk = k0 + kc;
            bool ok = (gr < mn_max) && (gk < k_max);
            const bf16* src = ok ? (g + (size_t)gr * ld + gk) : g;
            cp_async16(s + r * GEMM_LDK + kc, src, ok ? 16 : 0);
        }
    } else {
        // 32 rows(k) x 16 chunks = 512 chunks
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            int c = tid + i * GEMM_THREADS;
            int r = c >> 4, mc = (c & 15) * 8;
            int gk = k0 + r, gm = mn0 + mc;
            bool ok = (gk < k_max) && (gm < mn_max);
            const bf16* src = ok ? (g + (size_t)gk * ld + gm) : g;
            cp_async16(s + r * GEMM_LDMN + mc, src, ok ? 16 : 0);
        }
    }
}

// Epilogue concept:  void operator()(int row, int col, float v0, float v1) const   (col even; handles col, col+1)
//                    bounds are checked by the caller (row < M, col + 1 < N + 1).
template <int AMODE, int BMODE, class Epi>
__global__ void __launch_bounds__(GEMM_THREADS) gemm_bf16_kernel(const bf16* __restrict__ A, const bf16* __restrict__ B,
                                                                GemmShape sh, Epi epi) {
    pdl_wait();
    extern __shared__ __align__(16) unsigned char gemm_smem[];
    epi.prepare();
    bf16* sA = reinterpret_cast<bf16*>(gemm_smem);
    bf16* sB = sA + GEMM_STAGES * GEMM_TILE_ELEMS;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 2, wn = warp & 3;  // 2 x 4 warps ; warp tile 64 x 32
    const int m0 = blockIdx.y * GEMM_BM, n0 = blockIdx.x * GEMM_BN;
    const int kbeg = blockIdx.z * sh.k_per_split;
    const int kend = min(sh.K, kbeg + sh.k_per_split);
    const int nk = (kend - kbeg + GEMM_BK - 1) / GEMM_BK;
    // K-contiguous operands may read up to the next multiple of 8 (pad columns are finite, partner is zero-filled)
    const int kmax_contig = (sh.K + 7) & ~7;

    float acc[4][4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.f;

    auto load_stage = [&](int stage, int kt) {
        int k0 = kbeg + kt * GEMM_BK;
        gemm_load_tile<AMODE>(sA + stage * GEMM_TILE_ELEMS, A, sh.lda, m0, sh.M, k0,
                              AMODE == 0 ? min(kend, kmax_contig) : kend, tid);
        gemm_load_tile<BMODE>(sB + stage * GEMM_TILE_ELEMS, B, sh.ldb, n0, sh.N, k0,
                              BMODE == 0 ? min(kend, kmax_contig) : kend, tid);
    };

#pragma unroll
    for (int s = 0; s < GEMM_STAGES - 1; ++s) {
        if (s < nk) load_stage(s, s);
        cp_async_commit();
    }

    for (int kt = 0; kt < nk; ++kt) {
        cp_async_wait<GEMM_STAGES - 2>();
        __syncthreads();
        {
            int nxt = kt + GEMM_STAGES - 1;
            if (nxt < nk) load_stage(nxt % GEMM_STAGES, nxt);
            cp_async_commit();
        }
        const bf16* a_s = sA + (kt % GEMM_STAGES) * GEMM_TILE_ELEMS;
        const bf16* b_s = sB + (kt % GEMM_STAGES) * GEMM_TILE_ELEMS;
#pragma unroll
        for (int ks = 0; ks < GEMM_BK; ks += 16) {
            uint32_t af[4][4];
            uint32_t bfr[4][2];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                int mrow = wm * 64 + i * 16;
                if (AMODE == 0) {
                    ldsm_x4(af[i], a_s + (mrow + lane_a_row(lane)) * GEMM_LDK + ks + lane_a_col(lane));
                } else {
                    // stored [k][m]; transposed load: matrices (k0-7,m0-7),(k0-7,m8-15),(k8-15,m0-7),(k8-15,m8-15)
                    ldsm_x4_t(af[i], a_s + (ks + lane_b_row(lane)) * GEMM_LDMN + mrow + lane_b_col(lane));
                }
            }
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                int ncol = wn * 32 + j * 16;
                uint32_t r[4];
                if (BMODE == 0) {
                    ldsm_x4(r, b_s + (ncol + lane_b_row(lane)) * GEMM_LDK + ks + lane_b_col(lane));
                } else {
                    ldsm_x4_t(r, b_s + (ks + lane_a_row(lane)) * GEMM_LDMN + ncol + lane_a_col(lane));
                }
                bfr[2 * j][0] = r[0];
                bfr[2 * j][1] = r[1];
                bfr[2 * j + 1][0] = r[2];
                bfr[2 * j + 1][1] = r[3];
            }
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) mma_bf16(acc[i][j], af[i], bfr[j][0], bfr[j][1]);
        }
    }
    cp_async_wait<0>();

    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            int col = n0 + wn * 32 + j * 8 + 2 * t;
            int row = m0 + wm * 64 + i * 16 + g;
            if (col < sh.N) {
                if (row < sh.M) epi(row, col, acc[i][j][0], acc[i][j][1]);
                if (row + 8 < sh.M) epi(row + 8, col, acc[i][j][2], acc[i][j][3]);
            }
        }
    }
}

// ----------------------------------------------------------------------------- epilogues
// z = acc + bias ; write z (bf16) and act = dropout(silu(z)) (bf16).  [T, N]
struct EpiBiasSilu {
    const float* bias;
    bf16* z_out;
    bf16* act_out;
    int ld;
    Dropout drop;
    GRB_DEVINL void prepare() { drop.resolve(); }
    GRB_DEVINL void operator()(int row, int col, float v0, float v1) const {
        v0 += bias[col];
        v1 += bias[col + 1];
        size_t o = (size_t)row * ld + col;
        uint32_t zz = pack_bf16(v0, v1);
        *reinterpret_cast<uint32_t*>(z_out + o) = zz;
        float2 zr = unpack_bf16(zz);  // activation of the ROUNDED pre-activation (what the backward recomputes from)
        float a0 = siluf(zr.x), a1 = siluf(zr.y);
        drop.apply2(a0, a1, row, col);
        *reinterpret_cast<uint32_t*>(act_out + o) = pack_bf16(a0, a1);
    }
};
// acc + bias (no activation) -> bf16   (SASRec q/k/v projections)
struct EpiBiasBf16 {
    const float* bias;
    bf16* out;
    int ld;
    GRB_DEVINL void prepare() {}
    GRB_DEVINL void operator()(int row, int col, float v0, float v1) const {
        size_t o = (size_t)row * ld + col;
        *reinterpret_cast<uint32_t*>(out + o) = pack_bf16(v0 + bias[col], v1 + bias[col + 1]);
    }
};
// z = acc + bias ; write z and relu(z) w/ dropout   (SASRec fc1)
struct EpiBiasRelu {
    const float* bias;
    bf16* z_out;
    bf16* act_out;
    int ld;
    Dropout drop;
    GRB_DEVINL void prepare() { drop.resolve(); }
    GRB_DEVINL void operator()(int row, int col, float v0, float v1) const {
        v0 += bias[col];
        v1 += bias[col + 1];
        size_t o = (size_t)row * ld + col;
        uint32_t zz = pack_bf16(v0, v1);
        *reinterpret_cast<uint32_t*>(z_out + o) = zz;
        float2 zr = unpack_bf16(zz);
        float a0 = fmaxf(zr.x, 0.f), a1 = fmaxf(zr.y, 0.f);
        drop.apply2(a0, a1, row, col);
        *reinterpret_cast<uint32_t*>(act_out + o) = pack_bf16(a0, a1);
    }
};
// y = res + dropout(acc + bias) ; fp32 out (+ optional row mask multiply for SASRec)
struct EpiBiasResidual {
    const float* bias;
    const float* res;
    float* out;
    const float* row_scale;  // nullable: out *= row_scale[row]
    int ld;
    Dropout drop;
    GRB_DEVINL void prepare() { drop.resolve(); }
    GRB_DEVINL void operator()(int row, int col, float v0, float v1) const {
        size_t o = (size_t)row * ld + col;
        float2 r = *reinterpret_cast<const float2*>(res + o);
        float y0 = v0 + bias[col], y1 = v1 + bias[col + 1];
        drop.apply2(y0, y1, row, col);
        y0 += r.x;
        y1 += r.y;
        if (row_scale) {
            float s = row_scale[row];
            y0 *= s;
            y1 *= s;
        }
        *reinterpret_cast<float2*>(out + o) = make_float2(y0, y1);
    }
};
// g = dropmask(acc) * act'(z)  -> bf16   (ACT 0: silu, 1: relu)
template <int ACT>
struct EpiDAct {
    const bf16* z;
    bf16* out;
    int ld;
    Dropout drop;
    GRB_DEVINL void prepare() { drop.resolve(); }
    GRB_DEVINL void operator()(int row, int col, float v0, float v1) const {
        size_t o = (size_t)row * ld + col;
        float2 zz = unpack_bf16(*reinterpret_cast<const uint32_t*>(z + o));
        drop.apply2(v0, v1, row, col);
        float d0 = ACT == 0 ? dsiluf(zz.x) : (zz.x > 0.f ? 1.f : 0.f);
        float d1 = ACT == 0 ? dsiluf(zz.y) : (zz.y > 0.f ? 1.f : 0.f);
        *reinterpret_cast<uint32_t*>(out + o) = pack_bf16(v0 * d0, v1 * d1);
    }
};
// out = scale * acc (+ res) -> fp32
struct EpiF32 {
    float* out;
    const float* res;  // nullable
    int ld;
    float scale;
    GRB_DEVINL void prepare() {}
    GRB_DEVINL void operator()(int row, int col, float v0, float v1) const {
        size_t o = (size_t)row * ld + col;
        float y0 = v0 * scale, y1 = v1 * scale;
        if (res) {
            float2 r = *reinterpret_cast<const float2*>(res + o);
            y0 += r.x;
            y1 += r.y;
        }
        *reinterpret_cast<float2*>(out + o) = make_float2(y0, y1);
    }
};
// out += scale * acc   (split-K partial sums ; weight gradients accumulate into the flat grad buffer)
struct EpiAtomicF32 {
    float* out;
    int ld;
    float scale;
    GRB_DEVINL void prepare() {}
    GRB_DEVINL void operator()(int row, int col, float v0, float v1) const {
        size_t o = (size_t)row * ld + col;
        atomicAdd(out + o, v0 * scale);
        atomicAdd(out + o + 1, v1 * scale);
    }
};
// plain bf16 store
struct EpiBf16 {
    bf16* out;
    int ld;
    GRB_DEVINL void prepare() {}
    GRB_DEVINL void operator()(int row, int col, float v0, float v1) const {
        *reinterpret_cast<uint32_t*>(out + (size_t)row * ld + col) = pack_bf16(v0, v1);
    }
};
// plain fp32 store that tolerates an odd leading dimension (logits returned to the caller as [T, V+1] fp32)
struct EpiF32Scalar {
    float* out;
    int ld;
    int n;
    GRB_DEVINL void prepare() {}
    GRB_DEVINL void operator()(int row, int col, float v0, float v1) const {
        out[(size_t)row * ld + col] = v0;
        if (col + 1 < n) out[(size_t)row * ld + col + 1] = v1;
    }
};

template <int AMODE, int BMODE, class Epi>
inline cudaError_t launch_gemm(const bf16* A, const bf16* B, int M, int N, int K, int lda, int ldb, int splits,
                               const Epi& epi, cudaStream_t st) {
    GemmShape sh;
    sh.M = M;
    sh.N = N;
    sh.K = K;
    sh.lda = lda;
    sh.ldb = ldb;
    if (splits < 1) splits = 1;
    int kt = (K + GEMM_BK - 1) / GEMM_BK;
    int per = (kt + splits - 1) / splits;
    sh.k_per_split = per * GEMM_BK;
    splits = (kt + per - 1) / per;
    static bool attr_set = false;  // per template instantiation
    auto kern = gemm_bf16_kernel<AMODE, BMODE, Epi>;
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM_BYTES);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    dim3 grid((N + GEMM_BN - 1) / GEMM_BN, (M + GEMM_BM - 1) / GEMM_BM, splits);
    launch_k(kern, grid, GEMM_THREADS, GEMM_SMEM_BYTES, st, A, B, sh, epi);
    return cudaGetLastError();
}

}  // namespace grb
