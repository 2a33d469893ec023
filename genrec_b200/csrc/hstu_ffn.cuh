// genrec_b200 - the HSTU block's feed-forward as one wgmma kernel per direction (D = 64 or 128), built from tc_gemm.cuh's pieces.
//
//   forward : z1 = xn W1^T + b1 -> bf16 ; hact = drop(silu(z1)) -> bf16 ; y = x1 + drop(hact W2^T + b2) -> fp32
//   backward: dz1 = dropmask(dyb W2) * silu'(z1) -> bf16 ; dxn = dz1 W1 -> fp32
//
// The unfused path is two tc_gemm_kernel launches per direction, and the second one reads the [T, 4D] intermediate (hact or dz1)
// back from HBM.  Here a 128-row tile walks the 4D hidden dimension in 128-column chunks.  The chunk's first GEMM lands in
// registers, its epilogue writes the bf16 chunk into a 128B-swizzled [128 x 128] staging tile - the K-major SWIZZLE_128B layout of a
// wgmma A operand - and that tile is both TMA-stored to its [T, 4D] region and consumed in place as the A operand of the second
// GEMM, whose fp32 accumulators stay in registers across the chunks.  The staging tile is double-buffered, so the store of chunk c
// runs under the epilogue and the MMAs of chunk c + 1.
//
// Every value is bit-identical to the unfused kernels: the same m64n128k16 wgmma over the same k order (the second GEMM's k runs
// over the chunks in order, exactly the K loop of one GEMM over 4D), and the epilogues of TcEpiBiasAct<1>, TcEpiBiasResidual,
// TcEpiDAct<1> and TcEpiF32 restated per accumulator pair, with the same dropout keys (token row, column pair in the full width).
//
// Persistent kernel, one CTA per SM, 384 threads:
//   warp 0        : TMA producer (one elected lane) - the tile's resident A (xn / dyb), the weight chunks through a ring of
//                   FFN_STAGES 16 KB boxes and, backward, the saved z1 chunk (double-buffered)
//   warpgroups 1-2: consumers; warpgroup g owns rows 64 g .. 64 g + 63 of the tile: its wgmma, its epilogue (straight from the
//                   accumulator fragments) and its own bulk stores of its half of the staging tile, so the two never wait on each
//                   other inside a tile
// Both accumulators (64 + 64 fp32 per thread) are live through a chunk, so the producer warpgroup hands registers to the consumers.
//
// Where the time goes (cfg2 shape, T = 25,600, D = 128, H100 SXM at 700 W, per-phase clock64 stamps): a chunk is about 8,500 SM
// cycles, two thirds of them the epilogue (silu or silu', the dropout hash and the bf16 roundings of 64 elements per thread, bound
// by the SFU and by two warps per scheduler); its loads therefore go ahead of its shared-memory stores, all at once.  The forward's
// residual rows, read at the tile's end, are prefetched into L2 at its start and loaded into registers under the last chunk's MMAs.
// 200 tiles on 132 SMs make two rounds; splitting the work into 64-row units per warpgroup, so that the last round has one
// warpgroup per SM, measured slower (each warpgroup then needs its own weight ring).
#pragma once

#include "tc_gemm.cuh"

namespace grb {

constexpr int FFN_STAGES = 4;
constexpr int FFN_BOX = TC_TILE_BYTES;   // one [128 rows][64 bf16] 128B-swizzled box: 16 KB
constexpr int FFN_CHUNK = 128;           // hidden columns per chunk

template <int D>
struct FfnSmem {
    static constexpr int KD = D / 64;                          // k-blocks of the resident A (K = D)
    static constexpr int A_OFF = 0;                            // resident A: KD boxes
    static constexpr int RING_OFF = A_OFF + KD * FFN_BOX;      // weight ring: FFN_STAGES boxes
    static constexpr int H_OFF = RING_OFF + FFN_STAGES * FFN_BOX;   // staging of hact / dz1: 2 chunks of 2 boxes (128 x 128 each)
    static constexpr int Z_OFF = H_OFF + 4 * FFN_BOX;          // forward: z1 staging, 2 chunks ; backward: saved z1, 2 chunks
    static constexpr int BAR_OFF = Z_OFF + 4 * FFN_BOX;
    static constexpr int BYTES = BAR_OFF + 256 + 1024 /*align slack*/;
    static_assert(BYTES <= 227 * 1024, "shared memory budget of a Hopper block");
};

struct FfnArgs {
    int T;
    const float* b1;      // forward
    const float* b2;      // forward
    const float* x1;      // forward: residual [T, D]
    float* out;           // forward: y [T, D] ; backward: dxn [T, D]
    Dropout drop_hid;     // site 8 layer + 1: hact, and the dz1 mask
    Dropout drop_out;     // site 8 layer + 2: y (forward only)
};

GRB_DEVINL void setmaxnreg_dec40() { asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory"); }
GRB_DEVINL void setmaxnreg_inc232() { asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory"); }
// shared -> global tile store that puts the written lines first in line for L2 eviction: the forward's z1 and hact are next read by
// the backward, long after, and would otherwise push out the weights and the residual rows the kernel still reads
GRB_DEVINL void tma_store_2d_evict_first(const CUtensorMap* tmap, const void* smem_src, int c0, int c1, uint64_t policy) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%2, %3}], [%1], %4;" ::"l"(
                     reinterpret_cast<uint64_t>(tmap)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "l"(policy)
                 : "memory");
}

// byte offset of the bf16 pair (r, col), col even, in a [128 rows][128 cols] tile kept as two 128B-swizzled [128][64] boxes
GRB_DEVINL uint32_t ffn_pair_off(int r, int col) {
    return (uint32_t)((col >> 6) * FFN_BOX + r * 128 + ((((col & 63) >> 3) ^ (r & 7)) << 4) + (col & 7) * 2);
}
// all but the most recent bulk-store group of this thread have finished reading shared memory
GRB_DEVINL void tma_store_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }

// acc (+)= A[rows 64 g.., staging tile, nkb K-major boxes] * B[ring]: tc_mainloop with the accumulators carried over from the
// previous chunk (the first wgmma of the first chunk overwrites them, as the first one of a single GEMM's K loop does)
template <int B_MN>
GRB_DEVINL void ffn_mma_carry(float (&acc)[64], const unsigned char* sA, const unsigned char* sRing, uint64_t* full_bar, uint64_t* empty_bar,
                              int nkb, bool first, int g, int& stage, uint32_t& phase) {
    const bool leader = (threadIdx.x & 127) == 0;
    int prev = -1;
    for (int kb = 0; kb < nkb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t a_addr = smem_u32(sA + kb * FFN_BOX) + g * (FFN_BOX / 2);
        const uint32_t b_addr = smem_u32(sRing + stage * FFN_BOX);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_BK / 16; ++k) {
            const uint64_t ad = wgmma_desc(a_addr + k * 32, 16, 1024);
            const uint64_t bd = B_MN == 0 ? wgmma_desc(b_addr + k * 32, 16, 1024) : wgmma_desc(b_addr + k * 2048, FFN_BOX / 2, 1024);
            wgmma_m64n128k16<0, B_MN>(acc, ad, bd, (!first || kb > 0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();
        if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == FFN_STAGES) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (prev >= 0 && leader) mbar_arrive(&empty_bar[prev]);
}

// producer: one ring box (16 KB), once the consumers have released the slot
GRB_DEVINL void ffn_ring_wait(uint64_t* full_bar, uint64_t* empty_bar, int stage, uint32_t phase) {
    mbar_wait(&empty_bar[stage], phase ^ 1);
    mbar_expect_tx(&full_bar[stage], FFN_BOX);
}
GRB_DEVINL void ffn_ring_next(int& stage, uint32_t& phase) {
    if (++stage == FFN_STAGES) { stage = 0; phase ^= 1; }
}

// BWD = false: tmA = xn {64, 128}, tmW1 = W1 [4D][D] {64, 128}, tmW2 = W2 [D][4D] {64, 128}, tmZ / tmH = z1 / hact stores {64, 64}
// BWD = true : tmA = dyb {64, 128}, tmW1 = W1 as [K = 4D][N = D] {64, 64}, tmW2 = W2 as [K = D][N = 4D] {64, 64},
//              tmZ = saved z1 loads {64, 128}, tmH = dz1 stores {64, 64}
template <int D, bool BWD>
__global__ void __launch_bounds__(TC_THREADS, 1)
    hstu_ffn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmW2,
                    const __grid_constant__ CUtensorMap tmZ, const __grid_constant__ CUtensorMap tmH, FfnArgs a) {
    using S = FfnSmem<D>;
    constexpr int KD = S::KD, NC = 4 * D / FFN_CHUNK;
    extern __shared__ unsigned char ffn_smem_raw[];
    unsigned char* base = ffn_smem_raw + ((1024u - (smem_u32(ffn_smem_raw) & 1023u)) & 1023u);
    unsigned char* sA = base + S::A_OFF;
    unsigned char* sRing = base + S::RING_OFF;
    unsigned char* sH = base + S::H_OFF;
    unsigned char* sZ = base + S::Z_OFF;
    uint64_t* bars = reinterpret_cast<uint64_t*>(base + S::BAR_OFF);
    uint64_t* full_bar = bars;                        // [FFN_STAGES] TMA -> MMA
    uint64_t* empty_bar = bars + FFN_STAGES;          // [FFN_STAGES] MMA -> TMA (one arrive per consumer warpgroup)
    uint64_t* afull = bars + 2 * FFN_STAGES;          // resident A landed
    uint64_t* aempty = afull + 1;                     // both warpgroups' last first-GEMM of the tile has read it
    uint64_t* zfull = afull + 2;                      // [2] backward: saved z1 chunk landed
    uint64_t* zempty = afull + 4;                     // [2] backward: both warpgroups' epilogues have read it

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp == 0 && lane == 0) {
        tma_prefetch_desc(&tmA);
        tma_prefetch_desc(&tmW1);
        tma_prefetch_desc(&tmW2);
        for (int s = 0; s < FFN_STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 2);
        }
        mbar_init(afull, 1);
        mbar_init(aempty, 2);
        for (int s = 0; s < 2; ++s) {
            mbar_init(&zfull[s], 1);
            mbar_init(&zempty[s], 2);
        }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    a.drop_hid.resolve();
    a.drop_out.resolve();

    const int num_tiles = (a.T + TC_BM - 1) / TC_BM;
    if (warp < 4) {
        // ===================================================================== TMA producer
        setmaxnreg_dec40();
        if (warp == 0 && lane == 0) {
            int stage = 0;
            uint32_t phase = 0, aphase = 0, zphase = 0;
            int zb = 0;
            for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
                const int m0 = t * TC_BM;
                mbar_wait(aempty, aphase ^ 1);
                mbar_expect_tx(afull, KD * FFN_BOX);
                for (int kb = 0; kb < KD; ++kb) tma_load_2d(sA + kb * FFN_BOX, &tmA, kb * 64, m0, afull);
                aphase ^= 1;
                for (int c = 0; c < NC; ++c) {
                    const int h0 = c * FFN_CHUNK;
                    if constexpr (BWD) {
                        mbar_wait(&zempty[zb], zphase ^ 1);
                        mbar_expect_tx(&zfull[zb], 2 * FFN_BOX);
                        tma_load_2d(sZ + zb * 2 * FFN_BOX, &tmZ, h0, m0, &zfull[zb]);
                        tma_load_2d(sZ + zb * 2 * FFN_BOX + FFN_BOX, &tmZ, h0 + 64, m0, &zfull[zb]);
                        if (++zb == 2) { zb = 0; zphase ^= 1; }
                    }
                    // first GEMM's B: forward W1 rows h0.. (K-major) ; backward W2 columns h0.. (MN-major, two 64-wide boxes)
                    for (int kb = 0; kb < KD; ++kb) {
                        ffn_ring_wait(full_bar, empty_bar, stage, phase);
                        unsigned char* dst = sRing + stage * FFN_BOX;
                        if constexpr (BWD) {
                            tma_load_2d(dst, &tmW2, h0, kb * 64, &full_bar[stage]);
                            tma_load_2d(dst + FFN_BOX / 2, &tmW2, h0 + 64, kb * 64, &full_bar[stage]);
                        } else {
                            tma_load_2d(dst, &tmW1, kb * 64, h0, &full_bar[stage]);
                        }
                        ffn_ring_next(stage, phase);
                    }
                    // second GEMM's B over the chunk's 128 hidden k: forward W2 (K-major) ; backward W1 rows (MN-major)
                    for (int kb = 0; kb < 2; ++kb) {
                        ffn_ring_wait(full_bar, empty_bar, stage, phase);
                        unsigned char* dst = sRing + stage * FFN_BOX;
                        if constexpr (BWD) {
                            tma_load_2d(dst, &tmW1, 0, h0 + kb * 64, &full_bar[stage]);
                            tma_load_2d(dst + FFN_BOX / 2, &tmW1, 64, h0 + kb * 64, &full_bar[stage]);
                        } else {
                            tma_load_2d(dst, &tmW2, h0 + kb * 64, 0, &full_bar[stage]);
                        }
                        ffn_ring_next(stage, phase);
                    }
                }
            }
        }
    } else {
        // ===================================================================== consumers
        setmaxnreg_inc232();
        const int g = (warp >> 2) - 1;
        const int tw = threadIdx.x & 127, w = tw >> 5;
        const bool leader = tw == 0;
        const int rl = g * 64 + w * 16 + (lane >> 2);   // tile row of fragment rows i = 0 (+8 for i = 1)
        const int cl = 2 * (lane & 3);                   // column of fragment pair j: 8 j + cl
        int stage = 0, hb = 0;   // hb: this chunk's staging buffer (and, backward, its saved z1 buffer); it alternates every chunk
        uint32_t phase = 0, aphase = 0, zphase = 0;
        uint64_t evict_first = 0;
        if constexpr (!BWD) asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(evict_first));
        float acc1[64], acc2[64];
        for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
            const int m0 = t * TC_BM;
            if constexpr (!BWD) {
                // the tile's residual rows, read at its end, into L2 now: two threads per row, D / 64 lines of 128 B each
                const int pr = m0 + g * 64 + (tw >> 1);
                if (pr < a.T) {
#pragma unroll
                    for (int k = 0; k < D / 64; ++k)
                        asm volatile("prefetch.global.L2::evict_last [%0];" ::"l"(a.x1 + (size_t)pr * D + (tw & 1) * (D / 2) + k * 32));
                }
            }
            mbar_wait(afull, aphase);
            aphase ^= 1;
            for (int c = 0; c < NC; ++c) {
                const int h0 = c * FFN_CHUNK;
                tc_mainloop<0, BWD ? 1 : 0, FFN_STAGES, true>(acc1, sA, sRing, full_bar, empty_bar, 0, KD, g, stage, phase);
                if (c == NC - 1 && leader) mbar_arrive(aempty);
                if constexpr (BWD) mbar_wait(&zfull[hb], zphase);
                // this warpgroup's stores from staging buffer hb, two chunks back, have finished reading it (the previous chunk's may
                // still be in flight: they read the other buffer)
                if (leader) tma_store_wait_read1();
                wg_bar_sync(g);
                // The epilogue's loads (bias, saved z1) go ahead of its shared stores, all at once: interleaved, each load would wait
                // behind the previous pair's store.
                unsigned char* sHc = sH + hb * 2 * FFN_BOX;
                const unsigned char* sZc = sZ + hb * 2 * FFN_BOX;
                float2 pre[16][BWD ? 2 : 1];
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int col = 8 * j + cl;
                    if constexpr (BWD) {
#pragma unroll
                        for (int i = 0; i < 2; ++i) pre[j][i] = unpack_bf16(*reinterpret_cast<const uint32_t*>(sZc + ffn_pair_off(rl + 8 * i, col)));
                    } else {
                        pre[j][0] = make_float2(a.b1[h0 + col], a.b1[h0 + col + 1]);
                    }
                }
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const int col = 8 * j + cl;
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        const int r = rl + 8 * i;
                        const uint32_t row = (uint32_t)(m0 + r);
                        const uint32_t off = ffn_pair_off(r, col);
                        float v0 = acc1[4 * j + 2 * i], v1 = acc1[4 * j + 2 * i + 1];
                        if constexpr (BWD) {
                            // TcEpiDAct<1>
                            const float2 zz = pre[j][i];
                            a.drop_hid.apply2p(v0, v1, row, (uint32_t)(h0 + col) >> 1);
                            v0 *= dsiluf(zz.x);
                            v1 *= dsiluf(zz.y);
                            *reinterpret_cast<uint32_t*>(sHc + off) = pack_bf16(v0, v1);
                        } else {
                            // TcEpiBiasAct<1>
                            const float2 bb = pre[j][0];
                            const float z0 = v0 + bb.x, z1 = v1 + bb.y;
                            float w0 = siluf(bf16_round(z0)), w1 = siluf(bf16_round(z1));
                            a.drop_hid.apply2p(w0, w1, row, (uint32_t)(h0 + col) >> 1);
                            *reinterpret_cast<uint32_t*>(sZ + hb * 2 * FFN_BOX + off) = pack_bf16(z0, z1);
                            *reinterpret_cast<uint32_t*>(sHc + off) = pack_bf16(w0, w1);
                        }
                    }
                }
                fence_proxy_async();   // generic-proxy staging writes -> visible to the TMA stores and to wgmma
                wg_bar_sync(g);
                if constexpr (BWD) {
                    if (leader) mbar_arrive(&zempty[hb]);
                }
                if (leader) {
                    if (m0 + g * 64 < a.T) {
#pragma unroll
                        for (int b = 0; b < 2; ++b) {
                            const int so = hb * 2 * FFN_BOX + b * FFN_BOX + g * (FFN_BOX / 2);
                            if constexpr (BWD) {
                                tma_store_2d(&tmH, sH + so, h0 + 64 * b, m0 + g * 64);
                            } else {
                                tma_store_2d_evict_first(&tmH, sH + so, h0 + 64 * b, m0 + g * 64, evict_first);
                                tma_store_2d_evict_first(&tmZ, sZ + so, h0 + 64 * b, m0 + g * 64, evict_first);
                            }
                        }
                    }
                    tma_store_commit();
                }
                if constexpr (!BWD) {
                    // acc1 is free until the next tile: this thread's residual rows go into it, loaded under the last chunk's MMAs
                    if (c == NC - 1) {
#pragma unroll
                        for (int i = 0; i < 2; ++i) {
                            const int row = m0 + rl + 8 * i;
                            if (row >= a.T) continue;
#pragma unroll
                            for (int j = 0; j < D / 8; ++j) {
                                const float2 rr = *reinterpret_cast<const float2*>(a.x1 + (size_t)row * D + 8 * j + cl);
                                acc1[4 * j + 2 * i] = rr.x;
                                acc1[4 * j + 2 * i + 1] = rr.y;
                            }
                        }
                    }
                }
                ffn_mma_carry<BWD ? 1 : 0>(acc2, sHc, sRing, full_bar, empty_bar, 2, c == 0, g, stage, phase);
                if (++hb == 2) { hb = 0; zphase ^= 1; }
            }
            // tile end: y = x1 + drop(acc2 + b2) (TcEpiBiasResidual, no row scale) ; dxn = acc2 (TcEpiF32, scale 1, no residual)
            float2 b2v[D / 8];
            if constexpr (!BWD) {
#pragma unroll
                for (int j = 0; j < D / 8; ++j) b2v[j] = make_float2(a.b2[8 * j + cl], a.b2[8 * j + cl + 1]);
            }
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int row = m0 + rl + 8 * i;
                if (row >= a.T) continue;
                float* orow = a.out + (size_t)row * D;
#pragma unroll
                for (int j = 0; j < D / 8; ++j) {
                    const int col = 8 * j + cl;
                    float v0 = acc2[4 * j + 2 * i], v1 = acc2[4 * j + 2 * i + 1];
                    if constexpr (!BWD) {
                        float y0 = v0 + b2v[j].x, y1 = v1 + b2v[j].y;
                        a.drop_out.apply2p(y0, y1, (uint32_t)row, (uint32_t)col >> 1);
                        v0 = acc1[4 * j + 2 * i] + y0;
                        v1 = acc1[4 * j + 2 * i + 1] + y1;
                    }
                    *reinterpret_cast<float2*>(orow + col) = make_float2(v0, v1);
                }
            }
        }
        if (leader) tma_store_wait_read();   // smem must outlive this warpgroup's last bulk stores
    }
}

// forward: xn [T, D] bf16, W1 [4D, D], b1 [4D], W2 [D, 4D], b2 [D], x1 [T, D] fp32 -> z1, hact [T, 4D] bf16, y [T, D] fp32
template <int D>
inline cudaError_t launch_ffn_fwd(const bf16* xn, const bf16* w1, const float* b1, const bf16* w2, const float* b2, const float* x1, bf16* z1,
                                  bf16* hact, float* y, int T, const Dropout& drop_hid, const Dropout& drop_out, int num_sms, cudaStream_t st) {
    CUtensorMap tmA, tmW1, tmW2, tmZ, tmH;
    bool ok = make_tmap_bf16(&tmA, xn, T, D, D, 64, TC_BM);
    ok = ok && make_tmap_bf16(&tmW1, w1, 4 * D, D, D, 64, TC_BN);
    ok = ok && make_tmap_bf16(&tmW2, w2, D, 4 * D, 4 * D, 64, TC_BN);
    ok = ok && make_tmap_bf16(&tmZ, z1, T, 4 * D, 4 * D, 64, 64);
    ok = ok && make_tmap_bf16(&tmH, hact, T, 4 * D, 4 * D, 64, 64);
    if (!ok) return cudaErrorInvalidValue;
    const FfnArgs a{T, b1, b2, x1, y, drop_hid, drop_out};
    const int tiles = (T + TC_BM - 1) / TC_BM, grid = tiles < num_sms ? tiles : num_sms;
    return launch_k(hstu_ffn_kernel<D, false>, grid, TC_THREADS, FfnSmem<D>::BYTES, st, tmA, tmW1, tmW2, tmZ, tmH, a);
}
// backward: dyb [T, D] bf16, W2 [D, 4D], W1 [4D, D], saved z1 [T, 4D] -> dz1 [T, 4D] bf16, dxn [T, D] fp32
template <int D>
inline cudaError_t launch_ffn_bwd(const bf16* dyb, const bf16* w2, const bf16* w1, const bf16* z1, bf16* dz1, float* dxn, int T,
                                  const Dropout& drop_hid, int num_sms, cudaStream_t st) {
    CUtensorMap tmA, tmW1, tmW2, tmZ, tmH;
    bool ok = make_tmap_bf16(&tmA, dyb, T, D, D, 64, TC_BM);
    ok = ok && make_tmap_bf16(&tmW1, w1, 4 * D, D, D, 64, TC_BK);
    ok = ok && make_tmap_bf16(&tmW2, w2, D, 4 * D, 4 * D, 64, TC_BK);
    ok = ok && make_tmap_bf16(&tmZ, z1, T, 4 * D, 4 * D, 64, TC_BM);
    ok = ok && make_tmap_bf16(&tmH, dz1, T, 4 * D, 4 * D, 64, 64);
    if (!ok) return cudaErrorInvalidValue;
    const FfnArgs a{T, nullptr, nullptr, nullptr, dxn, drop_hid, make_dropout(0.f, 0, 0)};
    const int tiles = (T + TC_BM - 1) / TC_BM, grid = tiles < num_sms ? tiles : num_sms;
    return launch_k(hstu_ffn_kernel<D, true>, grid, TC_THREADS, FfnSmem<D>::BYTES, st, tmA, tmW1, tmW2, tmZ, tmH, a);
}

}  // namespace grb
