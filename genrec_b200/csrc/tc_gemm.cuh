// genrec_b200 - Hopper GEMM: TMA (cp.async.bulk.tensor, 128B swizzle) -> shared-memory ring (mbarrier pipeline) -> wgmma
// (fp32 accumulators in registers) -> shared-memory accumulator tile -> fused element-wise epilogue -> TMA stores.
//
//   C[M,N] (+)= A * opB(B)               bf16 operands, fp32 accumulate
//     A stored [M][K] (K contiguous)
//     B_MN = 0 : B stored [N][K] (K contiguous)        B_MN = 1 : B stored [K][N] (N contiguous)
//   Both majors map straight onto wgmma shared-memory descriptors (K-major / MN-major canonical SWIZZLE_128B layouts, the
//   MN-major ones through the instruction's transpose bits), so no operand is ever transposed in memory.  tc_mainloop also takes
//   an MN-major A, which the grouped weight-gradient GEMM (tc_tn_group.cuh) uses.
//
// Persistent kernel, one CTA per SM, 384 threads:
//   warp 0        : TMA producer (one elected lane)      - ring of TC_STAGES x (A 16 KB + B 16 KB)
//   warps 1-3     : idle (they complete the producer warpgroup so that the consumers are aligned warpgroups)
//   warpgroups 1-2: consumers; warpgroup g issues m64n128k16 wgmma for rows 64*g .. 64*g+63 of the 128 x 128 tile, parks the
//                   accumulators in shared memory and runs the epilogue on them: its warp w owns 32 rows and one 64-column
//                   half of the tile (the same row / column split for every epilogue functor below)
// Work item = one 128 x 128 output tile over the whole K.
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace grb {

constexpr int TC_EPI_WARPS = 8;    // 4 per consumer warpgroup: each converts TC_EPI_CPW 32-column chunks of 32 rows
constexpr int TC_EPI_CPW = 2;
constexpr int TC_BM = 128, TC_BN = 128, TC_BK = 64, TC_STAGES = 3, TC_THREADS = 128 + 32 * TC_EPI_WARPS;  // producer WG + 2 consumer WGs
constexpr int TC_TILE_BYTES = TC_BM * TC_BK * 2;  // 16 KB per operand per stage
constexpr int TC_STAGE_OUT_BYTES = 64 * 1024;   // epilogue staging: 2 x bf16 [128x128] or 1 x fp32 [128x128], 128B-swizzled boxes
constexpr int TC_ACC_BYTES = TC_BM * TC_BN * 4;  // fp32 accumulator tile
// 3 x 32 KB ring + 64 KB output staging + 64 KB accumulator tile = 224 KB of the 227 KB a Hopper block may use
constexpr int TC_SMEM_BYTES = 2 * TC_STAGES * TC_TILE_BYTES + TC_STAGE_OUT_BYTES + TC_ACC_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;

// ------------------------------------------------------------------------------------------------ PTX wrappers
GRB_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
GRB_DEVINL void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
GRB_DEVINL void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
GRB_DEVINL void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
GRB_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
GRB_DEVINL void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, int c0, int c1, uint64_t* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
                 : "memory");
}
// shared -> global tile store (bulk async group); rows/cols outside the tensor map's extents are clipped by the hardware
GRB_DEVINL void tma_store_2d(const CUtensorMap* tmap, const void* smem_src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(tmap)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}
GRB_DEVINL void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
GRB_DEVINL void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
GRB_DEVINL void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
GRB_DEVINL void tma_prefetch_desc(const CUtensorMap* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// the 128 threads of consumer warpgroup g (named barriers 2 and 3; 0 is __syncthreads)
GRB_DEVINL void wg_bar_sync(int g) { asm volatile("bar.sync %0, 128;" ::"r"(2 + g) : "memory"); }

GRB_DEVINL void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
GRB_DEVINL void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
GRB_DEVINL void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// D[64 x 128] (+)= A[smem desc, 64 x 16] * B[smem desc, 16 x 128]; TA / TB = 1: the operand is MN-major (transposed)
template <int TA, int TB>
GRB_DEVINL void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63}, %64, %65, p, 1, 1, %67, %68;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
}

// Shared-memory matrix descriptor, SWIZZLE_128B (sm_90 layout type 1).  Tile base must be 1024-byte aligned; `byte_off`
// selects the k-slice inside it.   K-major : rows of 128 B (64 bf16 along K), 8-row groups SBO = 1024 B apart.
//                                  MN-major: k-rows of 128 B (64 bf16 along MN), 8-k groups SBO = 1024 B apart, the next
//                                            64-wide MN block LBO bytes away.
GRB_DEVINL uint64_t wgmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= (uint64_t)1 << 62;  // SWIZZLE_128B
    return d;
}

// One consumer warpgroup's share of a work item: rows 64*g .. +63 of the 128 x 128 tile over k-blocks kb0 .. kb1-1 of the ring.
// Each stage is released to the producer once the wgmma reading it has retired (one MMA batch stays in flight).
template <int A_MN, int B_MN, int STAGES>
GRB_DEVINL void tc_mainloop(float (&acc)[64], const unsigned char* sA, const unsigned char* sB, uint64_t* full_bar, uint64_t* empty_bar,
                            int kb0, int kb1, int g, int& stage, uint32_t& phase) {
    const bool leader = (threadIdx.x & 127) == 0;
    int prev = -1;
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;   // the first wgmma overwrites them; this only ends their live range at the previous epilogue
    for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(sA + stage * TC_TILE_BYTES) + g * (TC_TILE_BYTES / 2);  // 64 rows (K-major) or one 64-wide M box
        const uint32_t b_addr = smem_u32(sB + stage * TC_TILE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) {
            // K-major: +32 B per 16-wide k-slice inside the 128 B swizzle row ; MN-major: +16 k-rows = 2048 B
            const uint64_t ad = A_MN == 0 ? wgmma_desc(a_addr + k * 32, 16, 1024) : wgmma_desc(a_addr + k * 2048, TC_TILE_BYTES / 2, 1024);
            const uint64_t bd = B_MN == 0 ? wgmma_desc(b_addr + k * 32, 16, 1024) : wgmma_desc(b_addr + k * 2048, TC_TILE_BYTES / 2, 1024);
            wgmma_m64n128k16<A_MN, B_MN>(acc, ad, bd, (kb > kb0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
}

// Accumulator tile in shared memory: fp32 [128 rows][128 cols], 16-byte chunk j of row r stored at chunk (j ^ (r & 7)), so that
// both the fragment stores below and the row-per-thread reads of the epilogue are free of bank conflicts.
GRB_DEVINL void tc_acc_store(float* sAcc, const float (&acc)[64], int g) {
    const int t = threadIdx.x & 127, w = t >> 5, lane = t & 31;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int r = g * 64 + w * 16 + (lane >> 2) + 8 * i;       // wgmma D fragment: row, column pair 8 j + 2 (lane % 4)
            const int c = 8 * j + 2 * (lane & 3);
            float* dst = sAcc + r * TC_BN + (((c >> 2) ^ (r & 7)) << 2) + (c & 3);
            *reinterpret_cast<float2*>(dst) = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
        }
    }
}
// columns c*32 .. c*32+31 of row r
GRB_DEVINL void tc_acc_load32(const float* sAcc, int r, int c, float (&v)[32]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float4 f = *reinterpret_cast<const float4*>(sAcc + r * TC_BN + (((c * 8 + j) ^ (r & 7)) << 2));
        v[4 * j] = f.x; v[4 * j + 1] = f.y; v[4 * j + 2] = f.z; v[4 * j + 3] = f.w;
    }
}

struct TcGemmShape {
    int M, N, K;
    int num_m, num_n;
    int kblocks_total;
};

// Epilogue concept:
//   static constexpr int kOut;   0: the functor stores by itself (odd strides)                signature (row, col0, v, nvalid)
//                                1: one bf16 output tile   2: two bf16 output tiles   3: one fp32 output tile
//                                   -> signature (row, col0, v /*in: acc, out: primary*/, w /*out: secondary*/, nvalid); the kernel
//                                      stages the tile in shared memory (128B swizzle) and writes it with TMA stores (tmC0 / tmC1).
//   void prepare();
template <int B_MN, class Epi>
__global__ void __launch_bounds__(TC_THREADS, 1)
    tc_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmC0,
                   const __grid_constant__ CUtensorMap tmC1, TcGemmShape sh, Epi epi) {
    extern __shared__ unsigned char tc_smem_raw[];
    // 1024-byte aligned operand ring, output staging, accumulator tile, then barriers
    unsigned char* base = tc_smem_raw + ((1024u - (smem_u32(tc_smem_raw) & 1023u)) & 1023u)   /* offset from the __shared__ array: keeps the shared address space (LDS / STS) */;
    unsigned char* sA = base;
    unsigned char* sB = base + TC_STAGES * TC_TILE_BYTES;
    unsigned char* sOut = base + 2 * TC_STAGES * TC_TILE_BYTES;
    float* sAcc = reinterpret_cast<float*>(sOut + TC_STAGE_OUT_BYTES);
    uint64_t* bars = reinterpret_cast<uint64_t*>(sOut + TC_STAGE_OUT_BYTES + TC_ACC_BYTES);
    uint64_t* full_bar = bars;                       // [TC_STAGES]  TMA -> MMA
    uint64_t* empty_bar = bars + TC_STAGES;          // [TC_STAGES]  MMA -> TMA (one arrive per consumer warpgroup)
    uint64_t* zempty_bar = bars + 2 * TC_STAGES;     // epilogue -> TMA: the auxiliary tile has been read (Epi::kAux)
    uint64_t* zfull_bar = bars + 2 * TC_STAGES + 1;  // TMA -> epilogue: auxiliary operand tile landed

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    epi.prepare();

    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmB);
        for (int s = 0; s < TC_STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 2);
        }
        mbar_init(zempty_bar, TC_EPI_WARPS);  // one arrive per epilogue warp
        mbar_init(zfull_bar, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();  // prologue above overlaps the previous kernel's tail

    const int num_work = sh.num_m * sh.num_n;

    if (warp < 4) {
        // ===================================================================== TMA producer
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0, zphase = 0;
            for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
                const int m0 = (w / sh.num_n) * TC_BM, n0 = (w % sh.num_n) * TC_BN;
                for (int kb = 0; kb < sh.kblocks_total; ++kb) {
                    mbar_wait(&empty_bar[stage], phase ^ 1);
                    mbar_expect_tx(&full_bar[stage], 2 * TC_TILE_BYTES);
                    unsigned char* a_dst = sA + stage * TC_TILE_BYTES;
                    unsigned char* b_dst = sB + stage * TC_TILE_BYTES;
                    const int k0 = kb * TC_BK;
                    tma_load_2d(a_dst, &tmA, k0, m0, &full_bar[stage]);                // box {64 k, 128 rows}
                    if (B_MN == 0) {
                        tma_load_2d(b_dst, &tmB, k0, n0, &full_bar[stage]);
                    } else {
                        tma_load_2d(b_dst, &tmB, n0, k0, &full_bar[stage]);
                        tma_load_2d(b_dst + TC_TILE_BYTES / 2, &tmB, n0 + 64, k0, &full_bar[stage]);
                    }
                    if (++stage == TC_STAGES) { stage = 0; phase ^= 1; }
                }
                if constexpr (Epi::kAux) {
                    // auxiliary element-wise operand of this tile -> the half of the staging buffer a single bf16 output leaves
                    // free, as soon as the epilogue of the previous tile has read it
                    mbar_wait(zempty_bar, zphase ^ 1);
                    unsigned char* z_dst = sOut + 32768;
                    mbar_expect_tx(zfull_bar, 32768);
                    tma_load_2d(z_dst, &tmC1, n0, m0, zfull_bar);                  // box {64 cols, 128 rows}
                    tma_load_2d(z_dst + 16384, &tmC1, n0 + 64, m0, zfull_bar);
                    zphase ^= 1;
                }
            }
        }
    } else {
        // ===================================================================== consumers: MMA + epilogue
        const int g = (warp >> 2) - 1;             // consumer warpgroup: tile rows 64 g .. 64 g + 63
        const int wi = warp & 3;
        const int sub = g * 2 + (wi & 1);          // 32-row slab of the tile this warp converts
        const int cq = wi >> 1;                    // which 64-column half of the tile this warp converts
        int stage = 0;
        uint32_t phase = 0, zphase = 0;
        float acc[64];
        for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
            const int m0 = (w / sh.num_n) * TC_BM, n0 = (w % sh.num_n) * TC_BN;
            tc_mainloop<0, B_MN, TC_STAGES>(acc, sA, sB, full_bar, empty_bar, 0, sh.kblocks_total, g, stage, phase);
            wg_bar_sync(g);                        // the previous tile's epilogue of this warpgroup has read sAcc
            tc_acc_store(sAcc, acc, g);
            wg_bar_sync(g);
            const int r = sub * 32 + lane;  // row inside the tile
            const int row = m0 + r;
            float pre[Epi::kPre ? TC_EPI_CPW : 1][Epi::kPre ? 32 : 1];
            if constexpr (Epi::kPre) {
#pragma unroll
                for (int ci = 0; ci < TC_EPI_CPW; ++ci) {
                    const int col0 = n0 + (cq * TC_EPI_CPW + ci) * 32;
                    const int nvalid = min(32, sh.N - col0);
                    if (row < sh.M && nvalid > 0) epi.preload(row, col0, nvalid, pre[ci]);
                }
            }
            if constexpr (Epi::kOut != 0) {
                if (lane == 0) tma_store_wait_read();   // this warp's store of the previous tile has finished reading its staging piece
                __syncwarp();
            }
            if constexpr (Epi::kAux) mbar_wait(zfull_bar, zphase);
#pragma unroll
            for (int ci = 0; ci < TC_EPI_CPW; ++ci) {
                const int c = cq * TC_EPI_CPW + ci;
                float v[32];
                tc_acc_load32(sAcc, r, c, v);
                const int col0 = n0 + c * 32;
                const int nvalid = min(32, sh.N - col0);
                if constexpr (Epi::kOut == 0) {
                    if (row < sh.M && nvalid > 0) epi(row, col0, v, nvalid);
                } else {
                    float w[32];
                    if constexpr (Epi::kAux) {
                        // this thread's 32 bf16 of the auxiliary tile (same 128B-swizzled box layout as the bf16 staging tile)
                        float zz[32];
                        const unsigned char* zsrc = sOut + 32768 + (c >> 1) * 16384 + r * 128;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const uint4 u = *reinterpret_cast<const uint4*>(zsrc + ((((c & 1) * 4 + j) ^ (r & 7)) << 4));
                            const float2 f0 = unpack_bf16(u.x), f1 = unpack_bf16(u.y), f2 = unpack_bf16(u.z), f3 = unpack_bf16(u.w);
                            zz[8 * j] = f0.x; zz[8 * j + 1] = f0.y; zz[8 * j + 2] = f1.x; zz[8 * j + 3] = f1.y;
                            zz[8 * j + 4] = f2.x; zz[8 * j + 5] = f2.y; zz[8 * j + 6] = f3.x; zz[8 * j + 7] = f3.y;
                        }
                        if (row < sh.M && nvalid > 0) epi(row, col0, v, w, nvalid, zz);
                    } else if constexpr (Epi::kPre) {
                        if (row < sh.M && nvalid > 0) epi(row, col0, v, w, nvalid, pre[ci]);
                    } else {
                        if (row < sh.M && nvalid > 0) epi(row, col0, v, w, nvalid);
                    }
                    if constexpr (Epi::kOut == 3) {
                        // fp32: box c = [128 rows][32 cols] = 128 B rows, 16-byte chunk j stored at (j ^ (r & 7))
                        unsigned char* dst = sOut + c * 16384 + r * 128;
#pragma unroll
                        for (int j = 0; j < 8; ++j)
                            *reinterpret_cast<float4*>(dst + ((j ^ (r & 7)) << 4)) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
                    } else {
                        // bf16: box h = [128 rows][64 cols]; this 32-column chunk covers 16-byte chunks (c&1)*4 .. +3 of box c>>1
                        unsigned char* dst = sOut + (c >> 1) * 16384 + r * 128;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            uint4 u;
                            u.x = pack_bf16(v[8 * j], v[8 * j + 1]); u.y = pack_bf16(v[8 * j + 2], v[8 * j + 3]);
                            u.z = pack_bf16(v[8 * j + 4], v[8 * j + 5]); u.w = pack_bf16(v[8 * j + 6], v[8 * j + 7]);
                            *reinterpret_cast<uint4*>(dst + ((((c & 1) * 4 + j) ^ (r & 7)) << 4)) = u;
                        }
                        if constexpr (Epi::kOut == 2) {
                            unsigned char* dst1 = dst + 32768;
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                uint4 u;
                                u.x = pack_bf16(w[8 * j], w[8 * j + 1]); u.y = pack_bf16(w[8 * j + 2], w[8 * j + 3]);
                                u.z = pack_bf16(w[8 * j + 4], w[8 * j + 5]); u.w = pack_bf16(w[8 * j + 6], w[8 * j + 7]);
                                *reinterpret_cast<uint4*>(dst1 + ((((c & 1) * 4 + j) ^ (r & 7)) << 4)) = u;
                            }
                        }
                    }
                }
            }
            if constexpr (Epi::kAux) {
                __syncwarp();
                if (lane == 0) mbar_arrive(zempty_bar);   // auxiliary tile read: the producer may load the next one
                zphase ^= 1;
            }
            if constexpr (Epi::kOut != 0) {
                // Every epilogue warp owns rows 32*sub .. +31 of the 64-column (bf16) / 2 x 32-column (fp32) slab cq of the staging
                // tile - a contiguous, swizzle-aligned 4 KB piece of each 128-row box - and stores it with its OWN bulk store (tensor-map
                // box = 32 rows): no CTA-wide barrier per tile.  Buffer reuse is guarded per warp by `wait_group.read 0` at the top of
                // the next tile.
                fence_proxy_async();   // generic-proxy smem writes -> visible to the TMA (async proxy)
                __syncwarp();
                if (lane == 0 && m0 + sub * 32 < sh.M) {
                    if constexpr (Epi::kOut == 3) {
#pragma unroll
                        for (int ci = 0; ci < TC_EPI_CPW; ++ci) {
                            const int c = cq * TC_EPI_CPW + ci;
                            if (n0 + c * 32 < sh.N) tma_store_2d(&tmC0, sOut + c * 16384 + sub * 4096, n0 + c * 32, m0 + sub * 32);
                        }
                    } else {
                        if (n0 + cq * 64 < sh.N) {
                            tma_store_2d(&tmC0, sOut + cq * 16384 + sub * 4096, n0 + cq * 64, m0 + sub * 32);
                            if constexpr (Epi::kOut == 2) tma_store_2d(&tmC1, sOut + 32768 + cq * 16384 + sub * 4096, n0 + cq * 64, m0 + sub * 32);
                        }
                    }
                }
                if (lane == 0) tma_store_commit();
            }
        }
        if (Epi::kOut != 0 && lane == 0) tma_store_wait_read();  // smem must outlive this warp's last bulk stores
    }
}

// ------------------------------------------------------------------------------------------------ row-chunk epilogues
GRB_DEVINL void store_bf16x32(bf16* dst, const float (&v)[32], int nvalid) {
    if (nvalid == 32 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            uint4 u;
            u.x = pack_bf16(v[8 * i], v[8 * i + 1]);
            u.y = pack_bf16(v[8 * i + 2], v[8 * i + 3]);
            u.z = pack_bf16(v[8 * i + 4], v[8 * i + 5]);
            u.w = pack_bf16(v[8 * i + 6], v[8 * i + 7]);
            reinterpret_cast<uint4*>(dst)[i] = u;
        }
    } else {
        for (int i = 0; i < nvalid; ++i) dst[i] = __float2bfloat16(v[i]);
    }
}
GRB_DEVINL void store_f32x32(float* dst, const float (&v)[32], int nvalid) {
    if (nvalid == 32 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) reinterpret_cast<float4*>(dst)[i] = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
    } else {
        for (int i = 0; i < nvalid; ++i) dst[i] = v[i];
    }
}
GRB_DEVINL void load_bf16x32(const bf16* src, float (&v)[32], int nvalid) {
    if (nvalid == 32 && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            uint4 u = reinterpret_cast<const uint4*>(src)[i];
            float2 a = unpack_bf16(u.x), b = unpack_bf16(u.y), c = unpack_bf16(u.z), d = unpack_bf16(u.w);
            v[8 * i] = a.x; v[8 * i + 1] = a.y; v[8 * i + 2] = b.x; v[8 * i + 3] = b.y;
            v[8 * i + 4] = c.x; v[8 * i + 5] = c.y; v[8 * i + 6] = d.x; v[8 * i + 7] = d.y;
        }
    } else {
        for (int i = 0; i < 32; ++i) v[i] = i < nvalid ? __bfloat162float(src[i]) : 0.f;
    }
}
GRB_DEVINL void load_f32x32(const float* src, float (&v)[32], int nvalid) {
    if (nvalid == 32 && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            float4 f = reinterpret_cast<const float4*>(src)[i];
            v[4 * i] = f.x; v[4 * i + 1] = f.y; v[4 * i + 2] = f.z; v[4 * i + 3] = f.w;
        }
    } else {
        for (int i = 0; i < 32; ++i) v[i] = i < nvalid ? src[i] : 0.f;
    }
}

// z = acc + bias -> bf16 ; act = dropout(ACT(z_rounded)) -> bf16      ACT 0: none (act_out unused), 1: silu, 2: relu
template <int ACT>
struct TcEpiBiasAct {
    static constexpr int kOut = ACT == 0 ? 1 : 2;   // tmC0 = z, tmC1 = act
    static constexpr bool kPre = false;
    static constexpr bool kAux = false;
    const float* bias;
    int ld;
    Dropout drop;
    GRB_DEVINL void prepare() { drop.resolve(); }
    GRB_DEVINL void operator()(int row, int col0, float (&v)[32], float (&w)[32], int nvalid) const {
        float bb[32];
        load_f32x32(bias + col0, bb, nvalid);
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            float zz = v[i] + bb[i];
            v[i] = zz;
            if (ACT != 0) {
                float zr = bf16_round(zz);
                w[i] = ACT == 1 ? siluf(zr) : fmaxf(zr, 0.f);
            }
        }
        if (ACT != 0) {
#pragma unroll
            for (int i = 0; i < 32; i += 2) drop.apply2p(w[i], w[i + 1], row, (col0 >> 1) + (i >> 1));
        }
    }
};
// y = res + dropout(acc + bias) (* row_scale) -> fp32
struct TcEpiBiasResidual {
    static constexpr int kOut = 3;
    static constexpr bool kPre = true;
    static constexpr bool kAux = false;
    const float* bias;
    const float* res;
    const float* row_scale;
    int ld;
    Dropout drop;
    GRB_DEVINL void prepare() { drop.resolve(); }
    GRB_DEVINL void preload(int row, int col0, int nvalid, float (&r)[32]) const { load_f32x32(res + (size_t)row * ld + col0, r, nvalid); }
    GRB_DEVINL void operator()(int row, int col0, float (&v)[32], float (&)[32], int nvalid, const float (&r)[32]) const {
        const float s = row_scale ? row_scale[row] : 1.f;
        float bb[32];
        load_f32x32(bias + col0, bb, nvalid);
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
            float y0 = v[i] + bb[i], y1 = v[i + 1] + bb[i + 1];
            drop.apply2p(y0, y1, row, (col0 >> 1) + (i >> 1));
            v[i] = (r[i] + y0) * s;
            v[i + 1] = (r[i + 1] + y1) * s;
        }
    }
};
// g = dropmask(acc) * ACT'(z) -> bf16
template <int ACT>
struct TcEpiDAct {
    static constexpr int kOut = 1;
    static constexpr bool kPre = false;
    static constexpr bool kAux = true;   // the saved pre-activation tile z[128 x 128] arrives by TMA (tensor map in the kernel's tmC1 slot)
    const bf16* z;
    int ld;
    Dropout drop;
    GRB_DEVINL void prepare() { drop.resolve(); }
    GRB_DEVINL void operator()(int row, int col0, float (&v)[32], float (&)[32], int nvalid, const float (&zz)[32]) const {
#pragma unroll
        for (int i = 0; i < 32; i += 2) {
            drop.apply2p(v[i], v[i + 1], row, (col0 >> 1) + (i >> 1));
            v[i] *= ACT == 1 ? dsiluf(zz[i]) : (zz[i] > 0.f ? 1.f : 0.f);
            v[i + 1] *= ACT == 1 ? dsiluf(zz[i + 1]) : (zz[i + 1] > 0.f ? 1.f : 0.f);
        }
    }
};
// out = scale * acc (+ res) -> fp32
struct TcEpiF32 {
    static constexpr int kOut = 3;
    static constexpr bool kPre = true;
    static constexpr bool kAux = false;
    const float* res;
    int ld;
    float scale;
    GRB_DEVINL void prepare() {}
    GRB_DEVINL void preload(int row, int col0, int nvalid, float (&y)[32]) const {
        if (res) load_f32x32(res + (size_t)row * ld + col0, y, nvalid);
    }
    GRB_DEVINL void operator()(int row, int col0, float (&v)[32], float (&)[32], int nvalid, const float (&y)[32]) const {
        if (res) {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = y[i] + v[i] * scale;
        } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] *= scale;
        }
    }
};
// exp(x) to ~1 ulp with FMA-pipe arithmetic only (the library is compiled with --use_fast_math, which would turn expf into the
// 2^-21-accurate ex2.approx path): Cody-Waite reduction x = n ln2 + r, |r| <= ln2 / 2, degree-6 polynomial, scale by 2^n.
GRB_DEVINL float exp_accurate(float x) {
    x = fminf(fmaxf(x, -87.f), 88.f);
    const float n = rintf(x * 1.44269504088896341f);
    float r = __fmaf_rn(n, -0.693145751953125f, x);            // ln2 high part (exact product for |n| < 2^10)
    r = __fmaf_rn(n, -1.42860682030941723e-6f, r);             // ln2 low part
    float p = 1.f / 720.f;
    p = __fmaf_rn(p, r, 1.f / 120.f);
    p = __fmaf_rn(p, r, 1.f / 24.f);
    p = __fmaf_rn(p, r, 1.f / 6.f);
    p = __fmaf_rn(p, r, 0.5f);
    p = __fmaf_rn(p, r, 1.f);
    p = __fmaf_rn(p, r, 1.f);
    return p * __int_as_float(((int)n + 127) << 23);
}
// out = ACT(res + acc + bias) + res2 -> fp32 : second pass of the split-bf16 GEMM (res = the sum of the five small cross terms;
// bias [N] and res2 [M, ld] nullable: the linear layers and the residual connection of the fp32-exact HSTU block)
template <int ACT>
struct TcEpiActResF32 {
    static constexpr int kOut = 3;
    static constexpr bool kPre = true;
    static constexpr bool kAux = false;
    const float* res;
    int ld;
    const float* bias;
    const float* res2;
    GRB_DEVINL void prepare() {}
    GRB_DEVINL void preload(int row, int col0, int nvalid, float (&y)[32]) const { load_f32x32(res + (size_t)row * ld + col0, y, nvalid); }
    GRB_DEVINL void operator()(int row, int col0, float (&v)[32], float (&)[32], int nvalid, const float (&y)[32]) const {
        float bb[32], rr[32];
        if (bias) load_f32x32(bias + col0, bb, nvalid);
        if (res2) load_f32x32(res2 + (size_t)row * ld + col0, rr, nvalid);
#pragma unroll
        for (int i = 0; i < 32; ++i) {
            float z = v[i] + y[i];
            if (bias) z += bb[i];
            z = ACT == 1 ? __fdiv_rn(z, 1.f + exp_accurate(-z)) : z;
            v[i] = res2 ? z + rr[i] : z;
        }
    }
};
// plain fp32 store, arbitrary leading dimension
struct TcEpiF32Plain {
    static constexpr int kOut = 0;
    static constexpr bool kPre = false;
    static constexpr bool kAux = false;
    float* out;
    int ld;
    GRB_DEVINL void prepare() {}
    GRB_DEVINL void operator()(int row, int col0, const float (&v)[32], int nvalid) const {
        store_f32x32(out + (size_t)row * ld + col0, v, nvalid);
    }
};

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                        const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                        CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_tmapEncodeTiled tmap_encoder() {
    static PFN_tmapEncodeTiled fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
    }
    return fn;
}

// 2-D row-major tensor [rows][cols] with leading dimension ld (elements); box = {box_cols (inner, 128 bytes), box_rows}
inline bool make_tmap(CUtensorMap* m, const void* base, bool fp32, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_cols, uint32_t box_rows) {
    PFN_tmapEncodeTiled enc = tmap_encoder();
    if (!enc) return false;
    const uint64_t esz = fp32 ? 4 : 2;
    if ((reinterpret_cast<uintptr_t>(base) & 15) || ((ld * esz) & 15)) return false;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {ld * esz};
    cuuint32_t box[2] = {box_cols, box_rows};
    cuuint32_t estr[2] = {1, 1};
    return enc(m, fp32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}
inline bool make_tmap_bf16(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_cols, uint32_t box_rows) {
    return make_tmap(m, base, false, rows, cols, ld, box_cols, box_rows);
}

// A: [M][K] ld=lda.   B: B_MN == 0 -> [N][K] ld=ldb ; B_MN == 1 -> [K][N] ld=ldb.
// out0 / out1: output tensors [M][N] with leading dimension ldo (bf16 for kOut 1/2, fp32 for kOut 3); unused for kOut 0.
template <int B_MN, class Epi>
inline cudaError_t launch_tc_gemm(const bf16* A, const bf16* B, int M, int N, int K, int lda, int ldb, const Epi& epi, void* out0, void* out1,
                                  int ldo, int num_sms, cudaStream_t st) {
    CUtensorMap tmA, tmB, tmC0, tmC1;
    bool ok = make_tmap_bf16(&tmA, A, M, K, lda, TC_BK, TC_BM);
    ok = ok && (B_MN == 0 ? make_tmap_bf16(&tmB, B, N, K, ldb, TC_BK, TC_BN) : make_tmap_bf16(&tmB, B, K, N, ldb, 64, TC_BK));
    if (Epi::kOut == 0) {
        tmC0 = tmA; tmC1 = tmA;
    } else if (Epi::kOut == 3) {
        ok = ok && make_tmap(&tmC0, out0, true, M, N, ldo, 32, 32);     // store boxes: 32 rows, one per epilogue warp
        tmC1 = tmC0;
    } else {
        ok = ok && make_tmap(&tmC0, out0, false, M, N, ldo, 64, 32);
        if (Epi::kOut == 2) ok = ok && make_tmap(&tmC1, out1, false, M, N, ldo, 64, 32);
        else tmC1 = tmC0;
    }
    if constexpr (Epi::kAux) {
        static_assert(Epi::kOut == 1, "the auxiliary tile lives in the half of the staging buffer a single bf16 output leaves free");
        ok = ok && make_tmap(&tmC1, epi.z, false, M, N, epi.ld, 64, TC_BM);
    }
    if (!ok) return cudaErrorInvalidValue;
    TcGemmShape sh;
    sh.M = M; sh.N = N; sh.K = K;
    sh.num_m = (M + TC_BM - 1) / TC_BM;
    sh.num_n = (N + TC_BN - 1) / TC_BN;
    sh.kblocks_total = (K + TC_BK - 1) / TC_BK;
    auto kern = tc_gemm_kernel<B_MN, Epi>;
    static bool attr_set_dev[64] = {false};
    int attr_dev = 0;
    cudaGetDevice(&attr_dev);
    bool& attr_set = attr_set_dev[attr_dev & 63];   // the attribute is per device
    if (!attr_set) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_BYTES);
        if (e != cudaSuccess) return e;
        attr_set = true;
    }
    int work = sh.num_m * sh.num_n;
    int grid = work < num_sms ? work : num_sms;
    launch_k(kern, grid, TC_THREADS, TC_SMEM_BYTES, st, tmA, tmB, tmC0, tmC1, sh, epi);
    return cudaGetLastError();
}

}  // namespace grb
