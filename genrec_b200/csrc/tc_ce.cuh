// genrec_b200 - fused tied-embedding logits + cross-entropy on wgmma: loss, d(loss)/d(x) and d(loss)/d(table) without ever
// writing a [tokens, classes] tensor.  D = 64 or 128 (the table rows fit one shared-memory tile).
//
//   ce_rows_kernel   (row-stationary, one CTA per 128 token rows): the token tile X [128 x D] stays in shared memory while the
//                    table streams through a TMA ring in 64-class tiles.  Sweep 1: S = X E^T (wgmma, register accumulators),
//                    online row maximum / exponent sum and the target logit -> per-row loss and the row's log2-domain shift.
//                    Sweep 2: S again, G = (softmax - onehot) / count in registers, converted in place to the bf16 A operand of
//                    dX += G E (wgmma with A from registers, the same table tile read MN-major) -> dX [T, D] fp32, written once.
//   ce_table_kernel  (class-stationary, one CTA per 64 classes): the table tile stays resident while the token tiles stream;
//                    S^T = E X^T, G^T from the saved row shifts, dE += G^T X, the two consumer warpgroups take alternate token
//                    tiles and their sums are added in a fixed order -> dE [C, D] += once per element.
// Every sum runs in a fixed order, so the results do not depend on timing.
#pragma once
#include "tc_gemm.cuh"

namespace grb {

// D[64 x 64] (+)= A[smem desc, K-major] * B[smem desc]; TB = 1: B is MN-major
template <int TB>
GRB_DEVINL void wgmma_m64n64k16_ss(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, %32, %33, p, 1, 1, 0, %35;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TB));
}
// D[64 x 64] (+)= A[registers, 64 x 16 bf16] * B[smem desc]; TB = 1: B is MN-major
template <int TB>
GRB_DEVINL void wgmma_m64n64k16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, %38;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate), "n"(TB));
}
// D[64 x 128] (+)= A[registers, 64 x 16 bf16] * B[smem desc]; TB = 1: B is MN-major
template <int TB>
GRB_DEVINL void wgmma_m64n128k16_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %69, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, {%64,%65,%66,%67}, %68, p, 1, 1, %70;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate), "n"(TB));
}

template <int D>
GRB_DEVINL void wgmma_rs_d(float (&d)[D / 2], const uint32_t (&a)[4], uint64_t bdesc) {
    if constexpr (D == 64) wgmma_m64n64k16_rs<1>(d, a, bdesc, 1u);
    else wgmma_m64n128k16_rs<1>(d, a, bdesc, 1u);
}

constexpr int CE_THREADS = 384;           // producer warpgroup + 2 consumer warpgroups
constexpr int CE_STAGES = 4;
constexpr float CE_L2E = 1.4426950408889634f;

struct CeArgs {
    const long long* tg;        // [T] targets (0 = ignored)
    const float* inv_count;     // device scalar: 1 / #(targets != 0)
    int T, C;
    float* dx;                  // [T, D] fp32 out (nullable: loss only)
    float* shift;               // [T] out of ce_rows_kernel, in of ce_table_kernel: log2(sum_c 2^(S_c log2e)) (the log2-domain lse)
    float* row_loss;            // [T] out
    float* dtable;              // [C, D] += (ce_table_kernel)
};

template <int D>
struct CeSmem {
    static constexpr int XB = D / 64;                  // 64-column boxes
    static constexpr int ROW_TILE = XB * 128 * 128;    // [128 rows][D] bf16
    static constexpr int CLS_TILE = XB * 64 * 128;     // [64 rows][D] bf16
    static constexpr int ROWS_BYTES = ROW_TILE + CE_STAGES * CLS_TILE + 1024 + 256;
    static constexpr int TABLE_BYTES = CLS_TILE + CE_STAGES * CLS_TILE + 1024 + 256;
};

// S[64 x 64] = A (64 rows of a K-major tile, D wide) * B^T (64 rows of a K-major tile); box b of A at a_addr + b * a_box
template <int D>
GRB_DEVINL void ce_scores(float (&S)[32], uint32_t a_addr, int a_box, uint32_t b_addr) {
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk)
        wgmma_m64n64k16_ss<0>(S, wgmma_desc(a_addr + (kk >> 2) * a_box + (kk & 3) * 32, 16, 1024),
                              wgmma_desc(b_addr + (kk >> 2) * 8192 + (kk & 3) * 32, 16, 1024), kk > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
}
// acc[64 x D] += G (registers, 64 x 64 along K) * B (a [64 k-rows][D] K-major tile read MN-major: N = D contiguous)
template <int D>
GRB_DEVINL void ce_accumulate(float (&acc)[D / 2], const float (&G)[32], uint32_t b_addr) {
    uint32_t a[4][4];
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
        a[kk][0] = pack_bf16(G[8 * kk], G[8 * kk + 1]);
        a[kk][1] = pack_bf16(G[8 * kk + 2], G[8 * kk + 3]);
        a[kk][2] = pack_bf16(G[8 * kk + 4], G[8 * kk + 5]);
        a[kk][3] = pack_bf16(G[8 * kk + 6], G[8 * kk + 7]);
    }
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) wgmma_rs_d<D>(acc, a[kk], wgmma_desc(b_addr + kk * 2048, 8192, 1024));
    wgmma_commit();
    wgmma_wait<0>();
}

template <int D>
__global__ void __launch_bounds__(CE_THREADS, 1)
    ce_rows_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmE, CeArgs a) {
    using SM = CeSmem<D>;
    extern __shared__ unsigned char ce_smem_raw[];
    unsigned char* base = ce_smem_raw + ((1024u - (smem_u32(ce_smem_raw) & 1023u)) & 1023u);
    unsigned char* sX = base;
    unsigned char* sE = base + SM::ROW_TILE;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sE + CE_STAGES * SM::CLS_TILE);
    uint64_t* full = bars;
    uint64_t* empty = bars + CE_STAGES;
    uint64_t* xfull = bars + 2 * CE_STAGES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row0 = blockIdx.x * 128;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmX);
        tma_prefetch_desc(&tmE);
        for (int s = 0; s < CE_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
        mbar_init(xfull, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    const int ntile = (a.C + 63) / 64;
    const int sweeps = a.dx ? 2 : 1;

    if (warp < 4) {
        if (warp == 0 && lane == 0) {
            mbar_expect_tx(xfull, SM::ROW_TILE);
            for (int b = 0; b < SM::XB; ++b) tma_load_2d(sX + b * 16384, &tmX, b * 64, row0, xfull);
            int stage = 0;
            uint32_t phase = 0;
            for (int sw = 0; sw < sweeps; ++sw)
                for (int j = 0; j < ntile; ++j) {
                    mbar_wait(&empty[stage], phase ^ 1);
                    mbar_expect_tx(&full[stage], SM::CLS_TILE);
                    for (int b = 0; b < SM::XB; ++b) tma_load_2d(sE + stage * SM::CLS_TILE + b * 8192, &tmE, b * 64, j * 64, &full[stage]);
                    if (++stage == CE_STAGES) { stage = 0; phase ^= 1; }
                }
        }
        return;
    }
    // consumer warpgroup g: tile rows 64 g .. 64 g + 63 ; this thread: rows r[0], r[1] = r[0] + 8, columns 8 j + 2 q + {0, 1}
    const int g = (warp >> 2) - 1, w = warp & 3, q = lane & 3;
    const bool leader = (threadIdx.x & 127) == 0;
    int row[2], tgt[2];
    float ic[2];
    const float inv = *a.inv_count;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        row[i] = row0 + 64 * g + 16 * w + (lane >> 2) + 8 * i;
        tgt[i] = row[i] < a.T ? (int)a.tg[row[i]] : 0;
        ic[i] = tgt[i] != 0 ? inv : 0.f;
    }
    mbar_wait(xfull, 0);
    const uint32_t xa = smem_u32(sX) + g * 8192;
    int stage = 0;
    uint32_t phase = 0;
    float m[2] = {-INFINITY, -INFINITY}, s[2] = {0.f, 0.f}, tl[2] = {0.f, 0.f};
    for (int j = 0; j < ntile; ++j) {
        mbar_wait(&full[stage], phase);
        float S[32];
        ce_scores<D>(S, xa, 16384, smem_u32(sE + stage * SM::CLS_TILE));
        if (leader) mbar_arrive(&empty[stage]);
        if (++stage == CE_STAGES) { stage = 0; phase ^= 1; }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            float mx = -INFINITY;
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int col = j * 64 + 8 * jj + 2 * q + c;
                    float& v = S[jj * 4 + i * 2 + c];
                    if (col >= a.C) v = -INFINITY;
                    if (col == tgt[i]) tl[i] = v;
                    mx = fmaxf(mx, v);
                }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
            const float mn = fmaxf(m[i], mx);
            float acc = s[i] * ex2_fast((m[i] - mn) * CE_L2E);
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                for (int c = 0; c < 2; ++c) acc += ex2_fast((S[jj * 4 + i * 2 + c] - mn) * CE_L2E);
            s[i] = acc;
            m[i] = mn;
        }
    }
    float shift[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        s[i] += __shfl_xor_sync(0xffffffffu, s[i], 1);
        s[i] += __shfl_xor_sync(0xffffffffu, s[i], 2);
        tl[i] += __shfl_xor_sync(0xffffffffu, tl[i], 1);
        tl[i] += __shfl_xor_sync(0xffffffffu, tl[i], 2);
        shift[i] = m[i] * CE_L2E + __log2f(s[i]);
        if (q == 0 && row[i] < a.T) {
            a.row_loss[row[i]] = tgt[i] != 0 ? (m[i] + __logf(s[i]) - tl[i]) * ic[i] : 0.f;
            a.shift[row[i]] = shift[i];
        }
    }
    if (!a.dx) return;
    float dx[D / 2];
#pragma unroll
    for (int k = 0; k < D / 2; ++k) dx[k] = 0.f;
    for (int j = 0; j < ntile; ++j) {
        mbar_wait(&full[stage], phase);
        float S[32];
        const uint32_t e_addr = smem_u32(sE + stage * SM::CLS_TILE);
        ce_scores<D>(S, xa, 16384, e_addr);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj)
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int col = j * 64 + 8 * jj + 2 * q + c;
                    float& v = S[jj * 4 + i * 2 + c];
                    float gv = col < a.C ? ex2_fast(v * CE_L2E - shift[i]) * ic[i] : 0.f;
                    if (col == tgt[i]) gv -= ic[i];
                    v = gv;
                }
        ce_accumulate<D>(dx, S, e_addr);
        if (leader) mbar_arrive(&empty[stage]);
        if (++stage == CE_STAGES) { stage = 0; phase ^= 1; }
    }
#pragma unroll
    for (int jj = 0; jj < D / 8; ++jj)
#pragma unroll
        for (int i = 0; i < 2; ++i)
            if (row[i] < a.T)
                *reinterpret_cast<float2*>(a.dx + (size_t)row[i] * D + 8 * jj + 2 * q) = make_float2(dx[jj * 4 + i * 2], dx[jj * 4 + i * 2 + 1]);
}

template <int D>
__global__ void __launch_bounds__(CE_THREADS, 1)
    ce_table_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmE, CeArgs a) {
    using SM = CeSmem<D>;
    extern __shared__ unsigned char ce_smem_raw[];
    unsigned char* base = ce_smem_raw + ((1024u - (smem_u32(ce_smem_raw) & 1023u)) & 1023u);
    unsigned char* sE = base;
    unsigned char* sX = base + SM::CLS_TILE;
    uint64_t* bars = reinterpret_cast<uint64_t*>(sX + CE_STAGES * SM::CLS_TILE);
    uint64_t* full = bars;
    uint64_t* empty = bars + CE_STAGES;
    uint64_t* efull = bars + 2 * CE_STAGES;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int cls0 = blockIdx.x * 64;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmX);
        tma_prefetch_desc(&tmE);
        for (int s = 0; s < CE_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
        mbar_init(efull, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    const int ntt = (a.T + 63) / 64;
    const int g = (warp >> 2) - 1, w = warp & 3, q = lane & 3;
    float acc[D / 2];
    if (warp < 4) {
        if (warp == 0 && lane == 0) {
            mbar_expect_tx(efull, SM::CLS_TILE);
            for (int b = 0; b < SM::XB; ++b) tma_load_2d(sE + b * 8192, &tmE, b * 64, cls0, efull);
            // token tile tt -> stage tt % CE_STAGES; consumer warpgroup tt % 2 owns it (CE_STAGES is even)
            for (int tt = 0; tt < ntt; ++tt) {
                const int stage = tt % CE_STAGES;
                mbar_wait(&empty[stage], ((tt / CE_STAGES) & 1) ^ 1);
                mbar_expect_tx(&full[stage], SM::CLS_TILE);
                for (int b = 0; b < SM::XB; ++b) tma_load_2d(sX + stage * SM::CLS_TILE + b * 8192, &tmX, b * 64, tt * 64, &full[stage]);
            }
        }
    } else {
        const bool leader = (threadIdx.x & 127) == 0;
        int cls[2];
#pragma unroll
        for (int i = 0; i < 2; ++i) cls[i] = cls0 + 16 * w + (lane >> 2) + 8 * i;
        const float inv = *a.inv_count;
#pragma unroll
        for (int k = 0; k < D / 2; ++k) acc[k] = 0.f;
        mbar_wait(efull, 0);
        const uint32_t ea = smem_u32(sE) + 0;
        for (int tt = g; tt < ntt; tt += 2) {
            const int stage = tt % CE_STAGES;
            // this thread's 16 token columns: shift, target, 1 / count
            float sh[16], icc[16];
            int tg[16];
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int t = tt * 64 + 8 * jj + 2 * q + c;
                    const bool ok = t < a.T;
                    tg[jj * 2 + c] = ok ? (int)a.tg[t] : 0;
                    sh[jj * 2 + c] = ok ? a.shift[t] : 0.f;
                    icc[jj * 2 + c] = tg[jj * 2 + c] != 0 ? inv : 0.f;
                }
            mbar_wait(&full[stage], (tt / CE_STAGES) & 1);
            const uint32_t x_addr = smem_u32(sX + stage * SM::CLS_TILE);
            float S[32];
            ce_scores<D>(S, ea + 0, 8192, x_addr);   // S^T: rows = this warpgroup's... all 64 classes, columns = 64 tokens
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        float& v = S[jj * 4 + i * 2 + c];
                        const int k = jj * 2 + c;
                        float gv = ex2_fast(v * CE_L2E - sh[k]) * icc[k];
                        if (cls[i] == tg[k]) gv -= icc[k];
                        v = gv;
                    }
            ce_accumulate<D>(acc, S, x_addr);
            if (leader) mbar_arrive(&empty[stage]);
        }
    }
    // warpgroup 2 hands its sum to warpgroup 1 through shared memory (the X ring is free by now); fixed order: wg1 + wg2
    float* red = reinterpret_cast<float*>(sX);
    asm volatile("bar.sync 1, 384;" ::: "memory");
    if (g == 1) {
#pragma unroll
        for (int k = 0; k < D / 2; ++k) red[(size_t)k * 128 + (threadIdx.x & 127)] = acc[k];
    }
    asm volatile("bar.sync 1, 384;" ::: "memory");
    if (g == 0) {
#pragma unroll
        for (int jj = 0; jj < D / 8; ++jj)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int c = cls0 + 16 * w + (lane >> 2) + 8 * i;
                const int k = jj * 4 + i * 2;
                const float v0 = acc[k] + red[(size_t)k * 128 + (threadIdx.x & 127)];
                const float v1 = acc[k + 1] + red[(size_t)(k + 1) * 128 + (threadIdx.x & 127)];
                if (c < a.C) {
                    float* dst = a.dtable + (size_t)c * D + 8 * jj + 2 * q;
                    atomicAdd(dst, v0);          // one add per element and launch
                    atomicAdd(dst + 1, v1);
                }
            }
    }
}

template <int D>
inline cudaError_t ce_set_smem() {
    static bool attr_set[64] = {false};
    int dev = 0;
    cudaGetDevice(&dev);
    if (attr_set[dev & 63]) return cudaSuccess;
    cudaError_t e = cudaFuncSetAttribute(ce_rows_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, CeSmem<D>::ROWS_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(ce_table_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, CeSmem<D>::TABLE_BYTES);
    if (e == cudaSuccess) attr_set[dev & 63] = true;
    return e;
}
// loss per row, shift per row and (a.dx != null) d loss / d xf
template <int D>
inline cudaError_t launch_tc_ce(const bf16* xf, const bf16* table, const CeArgs& a, cudaStream_t st) {
    CUtensorMap tmX, tmE;
    if (!make_tmap_bf16(&tmX, xf, a.T, D, D, 64, 128) || !make_tmap_bf16(&tmE, table, a.C, D, D, 64, 64)) return cudaErrorInvalidValue;
    cudaError_t e = ce_set_smem<D>();
    if (e != cudaSuccess) return e;
    launch_k(ce_rows_kernel<D>, (a.T + 127) / 128, CE_THREADS, CeSmem<D>::ROWS_BYTES, st, tmX, tmE, a);
    return cudaGetLastError();
}
// a.dtable += d loss / d table, from the shifts launch_tc_ce left
template <int D>
inline cudaError_t launch_ce_table(const bf16* xf, const bf16* table, const CeArgs& a, cudaStream_t st) {
    CUtensorMap tmX, tmE;
    if (!make_tmap_bf16(&tmX, xf, a.T, D, D, 64, 64) || !make_tmap_bf16(&tmE, table, a.C, D, D, 64, 64)) return cudaErrorInvalidValue;
    cudaError_t e = ce_set_smem<D>();
    if (e != cudaSuccess) return e;
    launch_k(ce_table_kernel<D>, (a.C + 63) / 64, CE_THREADS, CeSmem<D>::TABLE_BYTES, st, tmX, tmE, a);
    return cudaGetLastError();
}

}  // namespace grb
