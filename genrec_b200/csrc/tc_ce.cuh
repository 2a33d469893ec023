// genrec_b200 - fused tied-embedding logits + cross-entropy on wgmma: loss, d(loss)/d(x) and d(loss)/d(table) without ever
// writing a [tokens, classes] tensor.  D = 64 or 128 (the table rows fit one shared-memory tile).
//
//   ce_rows_kernel   (row-stationary, 128 token rows per unit): the token tile X [128 x D] stays in shared memory while the
//                    table streams through a TMA ring in 64-class tiles.  Sweep 1: S = X E^T (wgmma, register accumulators),
//                    online row maximum / exponent sum and the target logit -> per-row loss and the row's log2-domain shift.
//                    Sweep 2: S again, G = (softmax - onehot) / count in registers, converted in place to the bf16 A operand of
//                    dX += G E (wgmma with A from registers, the same table tile read MN-major) -> dX [T, D] fp32.
//   ce_table_kernel  (class-stationary, 64 classes per unit): the table tile stays resident while the token tiles stream;
//                    S^T = E X^T, G^T from the saved row shifts, dE += G^T X, the two consumer warpgroups take alternate token
//                    tiles and their sums are added in a fixed order -> dE [C, D] += once per element.
// Load balance without reordering a sum: each sweep is cut into segments (contiguous class tiles of a row tile, token tiles of a
// class tile), and a segment continues from the running sums (row maximum, exponent sums, target logit, the dX or dE
// accumulators) the segment before it left in global memory, so every row and class sees the same operations in the same order
// as one uninterrupted sweep, and the results are the same bits whatever the segment count.  Both kernels are persistent: one CTA
// per SM takes (segment, tile) units from a counter, segment-major, and waits only for the previous segment of its chain.  At
// 128 x 200 tokens and 12,102 classes on 132 SMs, 200 row tiles x 2 sweeps on whole-sweep units need 4 rounds where 3.03 would
// do, 190 class tiles 2 where 1.44 would do; ce_segments picks the counts from the shapes and the SM count only.
// The steps of a tile (shared-memory set-up, producer loads, lane coordinates, online-softmax step, row finish, the table pass's
// column metadata, warpgroup hand-over) are functions of their own below: the sampled-softmax head (tc_sampled_ce.cuh) is built from the same ones.
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
constexpr int CE_MAX_SEGMENTS = 8;

struct CeArgs {
    const long long* tg;        // [T] targets (0 = ignored)
    const float* inv_count;     // device scalar: 1 / #(targets != 0)
    int T, C;
    float* dx;                  // [T, D] fp32 out (nullable: loss only); between the segments of a row tile it holds the running sum
    float* shift;               // [T] out of ce_rows_kernel, in of ce_table_kernel: log2(sum_c 2^(S_c log2e)) (the log2-domain lse)
    float* row_loss;            // [T] out
    float* dtable;              // [C, D] += (ce_table_kernel)
    int rseg, tseg;             // segments of a row tile's class sweep, of a class tile's token sweep
    int* rsched;                // [1 + 2 * row tiles]: unit counter, then statistics / dX segments finished per row tile
    int* tsched;                // [1 + class tiles]: unit counter, then segments finished per class tile (both zeroed per launch)
    float* rcarry;              // [3][T][4] running row maximum, exponent sum and target logit of each lane (rseg > 1)
    float* tcarry;              // [class tiles][2][D / 2][128] running dE sums of the two consumer warpgroups (tseg > 1)
};

// The smallest segment count s <= min(CE_MAX_SEGMENTS, span) for which items * s units, one CTA per SM on `sms` SMs, leave at most
// 1/16 of their rounds' slots idle; when none does, the count with the fullest rounds (the smallest on a tie).
inline int ce_segments(int items, int span, int sms) {
    const int cap = span < CE_MAX_SEGMENTS ? span : CE_MAX_SEGMENTS;
    int best = 1;
    long long best_n = 0, best_slots = 1;
    for (int s = 1; s <= cap; ++s) {
        const long long n = (long long)items * s, slots = (n + sms - 1) / sms * sms;
        if (16 * n >= 15 * slots) return s;
        if (n * best_slots > best_n * slots) { best = s; best_n = n; best_slots = slots; }
    }
    return best;
}
// the row pass sweeps every row tile twice (statistics, then dX); the table pass sweeps every class tile once
inline int ce_row_segments(int T, int C, int sms) { return ce_segments(2 * ((T + 127) / 128), (C + 63) / 64, sms); }
inline int ce_table_segments(int T, int C, int sms) { return ce_segments((C + 63) / 64, (T + 63) / 64, sms); }

template <int D>
struct CeSmem {
    static constexpr int XB = D / 64;                  // 64-column boxes
    static constexpr int ROW_TILE = XB * 128 * 128;    // [128 rows][D] bf16
    static constexpr int CLS_TILE = XB * 64 * 128;     // [64 rows][D] bf16
    static constexpr int ROWS_BYTES = ROW_TILE + CE_STAGES * CLS_TILE + 1024 + 256;
    static constexpr int TABLE_BYTES = CLS_TILE + CE_STAGES * CLS_TILE + 1024 + 256;
};

// Both kernels are persistent: every CTA takes units from a counter, so a unit only ever waits for units taken before it, whose
// CTAs are running.  Barrier 1: the producer warp and both consumer warpgroups between units; barrier 2: the consumers.
GRB_DEVINL void ce_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }
// the consumers wait until `need` segments of their chain have finished
GRB_DEVINL void ce_wait_chain(const int* flag, int need) {
    if (threadIdx.x == 128) {
        int v;
        do asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
        while (v < need);
    }
    ce_bar(2, 256);
}
// the consumers' stores of this segment are visible: count it finished
GRB_DEVINL void ce_finish_segment(int* flag) {
    __threadfence();
    ce_bar(2, 256);
    if (threadIdx.x == 128) atomicAdd(flag, 1);
}

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

// A CTA's dynamic shared memory: the stationary tile (128 token rows in a row pass, 64 classes in a table pass), the ring of
// CE_STAGES streamed 64-row tiles, and their barriers.
struct CeCta {
    unsigned char* stat;        // the stationary tile, 1024-byte aligned
    unsigned char* ring;        // CE_STAGES tiles of CeSmem<D>::CLS_TILE bytes
    uint64_t *full, *empty;     // per ring stage: the tile has landed / its readers are done with it
    uint64_t* sfull;            // the stationary tile has landed
    unsigned char* tail;        // the first byte after the 256 bytes kept for the barriers
};
// Every thread of the CTA: carve the shared memory, let thread 0 prefetch the descriptors and initialise the barriers, and wait for
// the kernel before.  A stage is released by `empty_arrivals` consumer warpgroups: 2 in a row pass, where both read every
// streamed tile, 1 in a table pass, where they take alternate tiles.
template <int D>
GRB_DEVINL CeCta ce_cta_init(unsigned char* raw, int stat_bytes, int empty_arrivals, const CUtensorMap* tmX, const CUtensorMap* tmE) {
    CeCta cta;
    cta.stat = raw + ((1024u - (smem_u32(raw) & 1023u)) & 1023u);
    cta.ring = cta.stat + stat_bytes;
    cta.full = reinterpret_cast<uint64_t*>(cta.ring + CE_STAGES * CeSmem<D>::CLS_TILE);
    cta.empty = cta.full + CE_STAGES;
    cta.sfull = cta.full + 2 * CE_STAGES;
    cta.tail = cta.ring + CE_STAGES * CeSmem<D>::CLS_TILE + 256;
    if (threadIdx.x == 0) {
        tma_prefetch_desc(tmX);
        tma_prefetch_desc(tmE);
        for (int s = 0; s < CE_STAGES; ++s) { mbar_init(&cta.full[s], 1); mbar_init(&cta.empty[s], empty_arrivals); }
        mbar_init(cta.sfull, 1);
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();
    return cta;
}
// producer: rows row0 .. row0 + ROWS - 1 of tm into the stationary tile
template <int D, int ROWS>
GRB_DEVINL void ce_tile_load(const CeCta& cta, const CUtensorMap* tm, int row0) {
    mbar_expect_tx(cta.sfull, D / 64 * ROWS * 128);
    for (int b = 0; b < D / 64; ++b) tma_load_2d(cta.stat + b * ROWS * 128, tm, b * 64, row0, cta.sfull);
}
// producer: rows row0 .. row0 + 63 of tm into ring stage `stage`, once its readers have released it (`empty_parity`)
template <int D>
GRB_DEVINL void ce_ring_load(const CeCta& cta, const CUtensorMap* tm, int row0, int stage, uint32_t empty_parity) {
    mbar_wait(&cta.empty[stage], empty_parity);
    mbar_expect_tx(&cta.full[stage], CeSmem<D>::CLS_TILE);
    for (int b = 0; b < D / 64; ++b) tma_load_2d(cta.ring + stage * CeSmem<D>::CLS_TILE + b * 8192, tm, b * 64, row0, &cta.full[stage]);
}

// A consumer thread's place in the 64 x 64 accumulator of its warpgroup g (0, 1): S[4 j + 2 i + c] is tile row row(0, i),
// i = 0, 1, column 8 j + 2 q + c, j = 0 .. 7, c = 0, 1.
struct CeLane {
    int g, w, q, lane;
    bool leader;                // arrives on the ring's `empty` barriers for its warpgroup
    GRB_DEVINL int row(int base, int i) const { return base + 16 * w + (lane >> 2) + 8 * i; }
};
GRB_DEVINL CeLane ce_lane() {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    return CeLane{(warp >> 2) - 1, warp & 3, lane & 3, lane, (threadIdx.x & 127) == 0};
}

// One 64-column tile of the online softmax of this thread's row i (0, 1): the running maximum m is shared by the quad that holds
// the row, the exponent sum s is this lane's part.  S is final: masked columns hold -inf.
GRB_DEVINL void ce_softmax_step(const float (&S)[32], int i, float& m, float& s) {
    float mx = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int c = 0; c < 2; ++c) mx = fmaxf(mx, S[jj * 4 + i * 2 + c]);
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float mn = fmaxf(m, mx);
    float acc = s * ex2_fast((m - mn) * CE_L2E);
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int c = 0; c < 2; ++c) acc += ex2_fast((S[jj * 4 + i * 2 + c] - mn) * CE_L2E);
    s = acc;
    m = mn;
}
// The end of a row's sweep: the quad's exponent sums are added; returns the row's log2-domain shift, lse = log sum_c exp(S_c)
GRB_DEVINL float ce_row_finish(float m, float s, float& lse) {
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    lse = m + __logf(s);
    return m * CE_L2E + __log2f(s);
}

// A table pass thread's 16 token columns of token tile tt (column kq = 2 j + c is token 64 tt + 8 j + 2 q + c): target, the
// row's shift and 1 / count.  target(t) reads the target of token t < T; tokens past T and ignored tokens get weight 0.
struct CeCols {
    int tg[16];
    float sh[16], icc[16];
};
template <class Target>
GRB_DEVINL void ce_table_cols(CeCols& k, const CeLane& l, int tt, int T, const float* shift, float inv, Target target) {
#pragma unroll
    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const int t = tt * 64 + 8 * jj + 2 * l.q + c;
            const bool ok = t < T;
            k.tg[jj * 2 + c] = ok ? target(t) : 0;
            k.sh[jj * 2 + c] = ok ? shift[t] : 0.f;
            k.icc[jj * 2 + c] = k.tg[jj * 2 + c] != 0 ? inv : 0.f;
        }
}
// The end of a table pass: warpgroup 2 hands its sums to warpgroup 1 through shared memory (the ring is free by now).  After
// ce_wg_handover, warpgroup 1 stores acc[kk] + ce_wg_peer(cta, kk): always wg1 + wg2, a fixed order.
template <int D>
GRB_DEVINL void ce_wg_handover(const CeCta& cta, const CeLane& l, const float (&acc)[D / 2]) {
    float* red = reinterpret_cast<float*>(cta.ring);
    ce_bar(2, 256);                                // both warpgroups are done with the ring
    if (l.g == 1) {
#pragma unroll
        for (int kk = 0; kk < D / 2; ++kk) red[(size_t)kk * 128 + (threadIdx.x & 127)] = acc[kk];
    }
    ce_bar(2, 256);
}
GRB_DEVINL float ce_wg_peer(const CeCta& cta, int kk) { return reinterpret_cast<const float*>(cta.ring)[(size_t)kk * 128 + (threadIdx.x & 127)]; }

// Unit u: sweep u / (rseg R) (0: statistics, 1: dX), segment k = u / R % rseg, row tile u % R: the class tiles
// [k ntile / rseg, (k + 1) ntile / rseg) of that row tile, continuing from the running sums segment k - 1 left in global memory.
template <int D>
__global__ void __launch_bounds__(CE_THREADS, 1)
    ce_rows_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmE, CeArgs a) {
    using SM = CeSmem<D>;
    extern __shared__ unsigned char ce_smem_raw[];
    __shared__ int unit_slot[2];
    const CeCta cta = ce_cta_init<D>(ce_smem_raw, SM::ROW_TILE, 2, &tmX, &tmE);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp >= 1 && warp < 4) return;            // warp 0 produces (lane 0 issues the loads), warps 4..11 consume
    const int ntile = (a.C + 63) / 64, R = (a.T + 127) / 128, K = a.rseg;
    const int units = (a.dx ? 2 : 1) * K * R;
    const CeLane l = ce_lane();                    // consumer warpgroup g: tile rows 64 g .. 64 g + 63
    const int q = l.q;
    int stage = 0;                                 // the table ring runs on across units
    uint32_t phase = 0;
    for (int n = 0;; ++n) {
        if (threadIdx.x == 0) unit_slot[n & 1] = atomicAdd(a.rsched, 1);
        ce_bar(1, 288);
        const int u = unit_slot[n & 1];
        if (u >= units) break;
        const bool dxp = u >= K * R;
        const int k = u / R % K, rt = u % R, row0 = rt * 128;
        const int j0 = k * ntile / K, j1 = (k + 1) * ntile / K;
        int* sdone = a.rsched + 1 + rt;            // statistics segments finished for this row tile
        int* xdone = a.rsched + 1 + R + rt;        // dX segments finished
        if (warp == 0) {
            if (lane == 0) {
                ce_tile_load<D, 128>(cta, &tmX, row0);
                for (int j = j0; j < j1; ++j) {
                    ce_ring_load<D>(cta, &tmE, j * 64, stage, phase ^ 1);
                    if (++stage == CE_STAGES) { stage = 0; phase ^= 1; }
                }
            }
            __syncwarp();
            continue;
        }
        int row[2], tgt[2];
        float ic[2];
        const float inv = *a.inv_count;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            row[i] = l.row(row0 + 64 * l.g, i);
            tgt[i] = row[i] < a.T ? (int)a.tg[row[i]] : 0;
            ic[i] = tgt[i] != 0 ? inv : 0.f;
        }
        mbar_wait(cta.sfull, n & 1);
        const uint32_t xa = smem_u32(cta.stat) + l.g * 8192;
        if (!dxp) {
            if (k > 0) ce_wait_chain(sdone, k);
            float m[2] = {-INFINITY, -INFINITY}, s[2] = {0.f, 0.f}, tl[2] = {0.f, 0.f};
            const size_t plane = (size_t)a.T * 4;
#pragma unroll
            for (int i = 0; i < 2; ++i)
                if (k > 0 && row[i] < a.T) {
                    const size_t at = (size_t)row[i] * 4 + q;
                    m[i] = __ldcg(a.rcarry + at);
                    s[i] = __ldcg(a.rcarry + plane + at);
                    tl[i] = __ldcg(a.rcarry + 2 * plane + at);
                }
            for (int j = j0; j < j1; ++j) {
                mbar_wait(&cta.full[stage], phase);
                float S[32];
                ce_scores<D>(S, xa, 16384, smem_u32(cta.ring + stage * SM::CLS_TILE));
                if (l.leader) mbar_arrive(&cta.empty[stage]);
                if (++stage == CE_STAGES) { stage = 0; phase ^= 1; }
                // classes past C leave the softmax; the target's logit is kept
#pragma unroll
                for (int i = 0; i < 2; ++i) {
#pragma unroll
                    for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                        for (int c = 0; c < 2; ++c) {
                            const int col = j * 64 + 8 * jj + 2 * q + c;
                            float& v = S[jj * 4 + i * 2 + c];
                            if (col >= a.C) v = -INFINITY;
                            if (col == tgt[i]) tl[i] = v;
                        }
                    ce_softmax_step(S, i, m[i], s[i]);
                }
            }
            if (k + 1 < K) {
#pragma unroll
                for (int i = 0; i < 2; ++i)
                    if (row[i] < a.T) {
                        const size_t at = (size_t)row[i] * 4 + q;
                        a.rcarry[at] = m[i];
                        a.rcarry[plane + at] = s[i];
                        a.rcarry[2 * plane + at] = tl[i];
                    }
            } else {
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    float lse;
                    const float shift = ce_row_finish(m[i], s[i], lse);
                    tl[i] += __shfl_xor_sync(0xffffffffu, tl[i], 1);
                    tl[i] += __shfl_xor_sync(0xffffffffu, tl[i], 2);
                    if (q == 0 && row[i] < a.T) {
                        a.row_loss[row[i]] = tgt[i] != 0 ? (lse - tl[i]) * ic[i] : 0.f;
                        a.shift[row[i]] = shift;
                    }
                }
            }
            ce_finish_segment(sdone);
        } else {
            // rows past T: zero X rows and zero weights, so their G is 0 whatever the shift
            if (k > 0) ce_wait_chain(xdone, k);
            else ce_wait_chain(sdone, K);
            float shift[2];
#pragma unroll
            for (int i = 0; i < 2; ++i) shift[i] = row[i] < a.T ? __ldcg(a.shift + row[i]) : 0.f;
            float dx[D / 2];
#pragma unroll
            for (int jj = 0; jj < D / 8; ++jj)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    float2 v = make_float2(0.f, 0.f);
                    if (k > 0 && row[i] < a.T) v = __ldcg(reinterpret_cast<const float2*>(a.dx + (size_t)row[i] * D + 8 * jj + 2 * q));
                    dx[jj * 4 + i * 2] = v.x;
                    dx[jj * 4 + i * 2 + 1] = v.y;
                }
            for (int j = j0; j < j1; ++j) {
                mbar_wait(&cta.full[stage], phase);
                float S[32];
                const uint32_t e_addr = smem_u32(cta.ring + stage * SM::CLS_TILE);
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
                if (l.leader) mbar_arrive(&cta.empty[stage]);
                if (++stage == CE_STAGES) { stage = 0; phase ^= 1; }
            }
#pragma unroll
            for (int jj = 0; jj < D / 8; ++jj)
#pragma unroll
                for (int i = 0; i < 2; ++i)
                    if (row[i] < a.T)
                        *reinterpret_cast<float2*>(a.dx + (size_t)row[i] * D + 8 * jj + 2 * q) = make_float2(dx[jj * 4 + i * 2], dx[jj * 4 + i * 2 + 1]);
            ce_finish_segment(xdone);
        }
    }
}

// Unit u: segment k = u / NC of class tile u % NC: the token tiles [k ntt / tseg, (k + 1) ntt / tseg), continuing from the sums
// segment k - 1 left.  Consumer warpgroup g takes the token tiles tt = g (mod 2) of every segment.
template <int D>
__global__ void __launch_bounds__(CE_THREADS, 1)
    ce_table_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmE, CeArgs a) {
    using SM = CeSmem<D>;
    extern __shared__ unsigned char ce_smem_raw[];
    __shared__ int unit_slot[2];
    const CeCta cta = ce_cta_init<D>(ce_smem_raw, SM::CLS_TILE, 1, &tmX, &tmE);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp >= 1 && warp < 4) return;
    const int ntt = (a.T + 63) / 64, NC = (a.C + 63) / 64, K = a.tseg;
    const CeLane l = ce_lane();
    const int g = l.g, q = l.q;
    uint32_t pos = 0;                              // token tiles this CTA has streamed: the ring position of the unit's first tile
    for (int n = 0;; ++n) {
        if (threadIdx.x == 0) unit_slot[n & 1] = atomicAdd(a.tsched, 1);
        ce_bar(1, 288);
        const int u = unit_slot[n & 1];
        if (u >= K * NC) break;
        const int k = u / NC, ct = u % NC, cls0 = ct * 64;
        const int t0 = k * ntt / K, t1 = (k + 1) * ntt / K;
        int* done = a.tsched + 1 + ct;
        if (warp == 0) {
            if (lane == 0) {
                ce_tile_load<D, 64>(cta, &tmE, cls0);
                // ring position p -> stage p % CE_STAGES
                for (int tt = t0; tt < t1; ++tt) {
                    const uint32_t p = pos + (tt - t0);
                    ce_ring_load<D>(cta, &tmX, tt * 64, p % CE_STAGES, ((p / CE_STAGES) & 1) ^ 1);
                }
            }
            __syncwarp();
            pos += t1 - t0;
            continue;
        }
        const int cls[2] = {l.row(cls0, 0), l.row(cls0, 1)};
        const float inv = *a.inv_count;
        float acc[D / 2];
        float* carry = a.tcarry + ((size_t)ct * 2 + g) * (D / 2) * 128 + (threadIdx.x & 127);
        if (k > 0) ce_wait_chain(done, k);
#pragma unroll
        for (int kk = 0; kk < D / 2; ++kk) acc[kk] = k > 0 ? __ldcg(carry + (size_t)kk * 128) : 0.f;
        mbar_wait(cta.sfull, n & 1);
        const uint32_t ea = smem_u32(cta.stat);
        for (int tt = t0 + ((t0 ^ g) & 1); tt < t1; tt += 2) {
            const uint32_t p = pos + (tt - t0);
            const int stage = p % CE_STAGES;
            CeCols col;
            ce_table_cols(col, l, tt, a.T, a.shift, inv, [&](int t) { return (int)a.tg[t]; });
            mbar_wait(&cta.full[stage], (p / CE_STAGES) & 1);
            const uint32_t x_addr = smem_u32(cta.ring + stage * SM::CLS_TILE);
            float S[32];
            ce_scores<D>(S, ea, 8192, x_addr);     // S^T: rows = the 64 classes, columns = 64 tokens
#pragma unroll
            for (int jj = 0; jj < 8; ++jj)
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int c = 0; c < 2; ++c) {
                        float& v = S[jj * 4 + i * 2 + c];
                        const int kq = jj * 2 + c;
                        float gv = ex2_fast(v * CE_L2E - col.sh[kq]) * col.icc[kq];
                        if (cls[i] == col.tg[kq]) gv -= col.icc[kq];
                        v = gv;
                    }
            ce_accumulate<D>(acc, S, x_addr);
            if (l.leader) mbar_arrive(&cta.empty[stage]);
        }
        pos += t1 - t0;
        if (k + 1 < K) {
#pragma unroll
            for (int kk = 0; kk < D / 2; ++kk) carry[(size_t)kk * 128] = acc[kk];
            ce_finish_segment(done);
            continue;
        }
        ce_wg_handover<D>(cta, l, acc);
        if (g == 0) {
#pragma unroll
            for (int jj = 0; jj < D / 8; ++jj)
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int c = l.row(cls0, i);
                    const int kk = jj * 4 + i * 2;
                    const float v0 = acc[kk] + ce_wg_peer(cta, kk), v1 = acc[kk + 1] + ce_wg_peer(cta, kk + 1);
                    if (c < a.C) {
                        float* dst = a.dtable + (size_t)c * D + 8 * jj + 2 * q;
                        atomicAdd(dst, v0);          // one add per element and launch
                        atomicAdd(dst + 1, v1);
                    }
                }
        }
    }
}

// loss per row, shift per row and (a.dx != null) d loss / d xf, on at most `ctas` CTAs
template <int D>
inline cudaError_t launch_tc_ce(const bf16* xf, const bf16* table, const CeArgs& a, int ctas, cudaStream_t st) {
    CUtensorMap tmX, tmE;
    if (!make_tmap_bf16(&tmX, xf, a.T, D, D, 64, 128) || !make_tmap_bf16(&tmE, table, a.C, D, D, 64, 64)) return cudaErrorInvalidValue;
    const int R = (a.T + 127) / 128, units = (a.dx ? 2 : 1) * a.rseg * R;
    const cudaError_t e = cudaMemsetAsync(a.rsched, 0, (size_t)(1 + 2 * R) * sizeof(int), st);
    if (e != cudaSuccess) return e;
    return launch_k(ce_rows_kernel<D>, units < ctas ? units : ctas, CE_THREADS, CeSmem<D>::ROWS_BYTES, st, tmX, tmE, a);
}
// a.dtable += d loss / d table, from the shifts launch_tc_ce left, on at most `ctas` CTAs
template <int D>
inline cudaError_t launch_ce_table(const bf16* xf, const bf16* table, const CeArgs& a, int ctas, cudaStream_t st) {
    CUtensorMap tmX, tmE;
    if (!make_tmap_bf16(&tmX, xf, a.T, D, D, 64, 64) || !make_tmap_bf16(&tmE, table, a.C, D, D, 64, 64)) return cudaErrorInvalidValue;
    const int NC = (a.C + 63) / 64, units = a.tseg * NC;
    const cudaError_t e = cudaMemsetAsync(a.tsched, 0, (size_t)(1 + NC) * sizeof(int), st);
    if (e != cudaSuccess) return e;
    return launch_k(ce_table_kernel<D>, units < ctas ? units : ctas, CE_THREADS, CeSmem<D>::TABLE_BYTES, st, tmX, tmE, a);
}

}  // namespace grb
