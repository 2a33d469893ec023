// genrec_b200 - cached incremental HSTU inference: append a chunk of items to a per-user K | V cache and run the chunk's
// rows through the attention against everything cached so far.
//
// Cache (per layer): kv [B, cap, 2D] bf16, row p of user b = K | V of the user's p-th item (items, not slots: pads are
// compacted away).  timestamps [B, cap] int64, lengths [B] int32, overflow [B] uint8 are shared by all layers.
//
// A valid chunk row i of user b sits at cache position p_i and attends to the keys [0, p_i] of its own user:
//   O_i = sum_{j <= p_i} silu(Q_i . K_j + Wpos[pb(p_i - j), h] + Wtime[tb(|ts_i - ts_j|), h]) V_j
// which is row i of the full forward (attn_hstu.cuh) whenever the history is left-padded: causal attention never looks
// right, and HSTU's biases depend on i - j and |ts_i - ts_j| only, so the amount of left padding cannot change a valid row.
// Time buckets are computed on the fly by time_bucket_dev with the same thresholds as hstu_bias_index_kernel (no [n, cap]
// index matrix), and silu(S) is rounded to bf16 before the A.V product as in hstu_attn_fwd_kernel.
//
// Parallelism: keys are split across CTAs (grid.x) so that one new item per user still fills the GPU.  Without a softmax
// the split partials combine by plain summation; each CTA stores its fp32 partial and hstu_extend_combine_kernel adds them
// in split order, so the result is the same from run to run.
//
// Paged pool: the same kernels serve a pool of K | V pages shared by many users.  Row b of a call belongs to user users[b]
// (any distinct subset of the pool's users), and item p of user u lives in page page_table[u, p / page_size] at row
// p % page_size.  The dense cache above is the degenerate pool: page_size = cap, page b belongs to user b, users = 0 .. B-1,
// which is what a null page table and a null user list stand for.  A page holds a whole number of 64-key tiles, so no key
// tile of the attention straddles two pages.  hstu_pool_alloc_kernel hands out the pages a call needs (one CTA, in row order,
// so the outcome of running out is deterministic) and hstu_pool_release_kernel gives a user's pages back.
#pragma once
#include "attn_hstu.cuh"

namespace grb {

// Where item p of user u is stored: row pg.row(u, p) of the [pages * page_size] rows of K | V (and of timestamps).
struct KvPages {
    const int* page_table;   // [users, pt_ld] page of each page_size items ; null: the dense cache (page u, page_size = capacity)
    int pt_ld, page_size;
    GRB_DEVINL size_t row(int u, int p) const {
        return page_table ? (size_t)page_table[(size_t)u * pt_ld + p / page_size] * page_size + p % page_size
                          : (size_t)u * page_size + p;
    }
};

// One warp per chunk row b of user u = users[b] (b without a user list).  pos[b, r] = len[u] + (valid rows of the chunk before
// r) for a valid row (id != 0), -1 for a pad and for an item that does not fit in the user's room (dropped; overflow[u] = 1).
// The room is room[b] (the pool: what the allocation left the user, -1 = a rejected row, treated as all padding) or `cap`
// without a room list.  The chunk's timestamps are written into the cache, len[u] becomes min(len[u] + valid, room) and
// last_row[b] is the chunk row of the user's last valid item, or -1.
// JAGGED (a packed chunk of T token rows, n = max_len): sequence b is the token rows of seq_span(offsets, T, n, b), ids / ts / pos
// are [T], and last_row[b] is the token row of the user's last valid item.  The caller sets pos to -1 beforehand: rows in no
// sequence (idle rows) are not visited.
template <bool JAGGED>
__global__ void __launch_bounds__(128) hstu_cache_append_kernel(const long long* __restrict__ ids, const long long* __restrict__ ts,
                                                                const long long* __restrict__ users, const int* __restrict__ room, int B,
                                                                int n, int cap, KvPages pg, long long* __restrict__ cache_ts,
                                                                int* __restrict__ len, uint8_t* __restrict__ overflow, int* __restrict__ pos,
                                                                int* __restrict__ last_row, const long long* __restrict__ offsets, int T) {
    pdl_wait();
    const int b = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= B) return;
    long long tok0 = 0;
    int rows = n;
    if constexpr (JAGGED) seq_span(offsets, T, n, b, tok0, rows);
    auto at = [&](int r) { return JAGGED ? (size_t)tok0 + r : (size_t)b * n + r; };   // the token row of row r of the sequence
    const int lim = room ? room[b] : cap;
    if (lim < 0) {
        for (int r = lane; r < rows; r += 32) pos[at(r)] = -1;
        if (lane == 0) last_row[b] = -1;
        return;
    }
    const int u = users ? (int)users[b] : b;
    const int base = len[u];
    int count = 0, last = -1;
    for (int r0 = 0; r0 < rows; r0 += 32) {
        const int r = r0 + lane;
        const bool valid = r < rows && ids[at(r)] != 0;
        const unsigned m = __ballot_sync(0xffffffffu, valid);
        const int q = base + count + __popc(m & ((1u << lane) - 1u));
        if (r < rows) {
            int p = -1;
            if (valid && q < lim) {
                p = q;
                cache_ts[pg.row(u, q)] = ts ? ts[at(r)] : 0;
            }
            pos[at(r)] = p;
        }
        if (m) last = r0 + 31 - __clz((int)m);
        count += __popc(m);
    }
    if (lane == 0) {
        const long long total = (long long)base + count;
        len[u] = total > lim ? lim : (int)total;
        if (total > lim) overflow[u] = 1;
        last_row[b] = JAGGED && last >= 0 ? (int)tok0 + last : last;
    }
}

// The sequence b of a packed batch whose rows seq_span(offsets, T, L, b) hold token row `row`, or -1 for an idle row: a binary
// search for the last b with offsets[b] <= row, then a check against that sequence's clamped span (a malformed device offsets
// gives some sequence or -1, never a row outside the span).
GRB_DEVINL int jagged_seq_of(const long long* offsets, int B, int T, int L, int row) {
    int lo = 0, hi = B - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (offsets[mid] <= row) lo = mid;
        else hi = mid - 1;
    }
    long long tok0;
    int len;
    seq_span(offsets, T, L, lo, tok0, len);
    return row >= tok0 && row < tok0 + len ? lo : -1;
}

// K | V row of every chunk row with pos >= 0 into the cache row of (users[b], pos): [0, D) = K, [D, 2D) = V.
// P = [U | V | Q | K] [B*n, 4D] bf16.  One thread per 16-byte piece.  JAGGED (P [T, 4D] of B sequences, n = max_len): the row's
// sequence comes from jagged_seq_of, searched only for rows that have a position.
template <bool JAGGED>
__global__ void __launch_bounds__(256) hstu_kv_scatter_kernel(const bf16* __restrict__ P, const int* __restrict__ pos,
                                                              const long long* __restrict__ users, int T, int n, int D, KvPages pg,
                                                              bf16* __restrict__ kv, const long long* __restrict__ offsets, int B) {
    pdl_wait();
    const int per_row = 2 * D / 8;
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)T * per_row) return;
    const int row = (int)(idx / per_row), c = (int)(idx % per_row) * 8;   // column of the cache row
    const int p = pos[row];
    if (p < 0) return;
    const int b = JAGGED ? jagged_seq_of(offsets, B, T, n, row) : row / n;
    if (JAGGED && b < 0) return;
    const int u = users ? (int)users[b] : b;
    const int src = c < D ? 3 * D + c : c;                                // K = P[:, 3D:4D) ; V = P[:, D:2D)
    *reinterpret_cast<uint4*>(kv + pg.row(u, p) * 2 * D + c) = *reinterpret_cast<const uint4*>(P + (size_t)row * 4 * D + src);
}

struct HstuExtendArgs {
    const bf16* q; int ldq;            // chunk queries, [B * n] rows (P + 2D, ld 4D)
    const bf16* kv;                    // this layer's K | V rows [pages * page_size, 2D]
    const long long* ts;               // [pages * page_size] cache timestamps
    const long long* users;            // [B] user of each chunk row ; null: row b is user b
    KvPages pg;
    const int* pos;                    // [B * n] cache position of each chunk row, -1 = none
    const uint8_t* pos_bucket;         // [cap] bucket of delta = p_i - j ; null: every delta uses the single live row of bias.wpos
    const long long* thr;              // [65] time-bucket thresholds
    HstuBiasArgs bias;                 // wpos / wtime / npos / ntime (bias_index unused)
    int B, n, H, D, cap;               // cap: most items a user can hold
    int split;                         // keys per CTA, a multiple of ATT_BLK ; grid.x = ceil(cap / split)
    float* part;                       // [grid.x, B * n, D] fp32 partial outputs ; a packed chunk: [grid.x, T, D]
    const long long* offsets;          // null: a padded [B, n] chunk ; else sequence b is token rows seq_span(offsets, T, n, b)
    int T;                             // token rows of a packed chunk (n = max_len)
};

template <int DH>
struct ExtSmem {
    static constexpr int LD = DH + 8;
    bf16 q[ATT_BLK * LD];
    bf16 kv[2][2][ATT_BLK * LD];       // [buffer][K, V]
    long long ts[2][ATT_BLK];          // [buffer] key timestamps
    long long thr[ATT_MAX_BUCKETS + 1];
    int pmax;
};
// dynamic tail: float wcomb[npos * 64 + 1] (att_build_table) ; JAGGED: then, 16-byte aligned, the sequence's first token row
__host__ __device__ inline size_t ext_table_bytes(int npos) { return ((size_t)(npos * 64 + 1) * 4 + 15) / 16 * 16; }

// grid (ceil(cap / split), H, B * ceil(n / 64)), 128 threads: 64 chunk rows of one user and head against the keys
// [split * x, split * (x + 1)) of the user's cache.  Tiles that lie beyond every row's position are skipped.  JAGGED: the
// tile's rows are those of sequence b from its first token row, and a tile past the sequence's end exits.
// CTAs per SM of the padded instantiation (ptxas -v registers, 128 threads), which the packed one is held to: its sequence's
// first row and length come from a load, not from the launch, and ptxas otherwise spends more registers on them and loses an
// SM slot.  0 (no floor) where the floor would spill: the packed kernel has the padded kernel's occupancy without it at dh 32,
// and loses one CTA per SM at dh 64 (130 registers against 128).
template <int DH, bool UNIFORM, bool TIMED>
constexpr int ext_jagged_min_blocks() {
    return DH == 32 ? (UNIFORM ? (TIMED ? 5 : 0) : (TIMED ? 3 : 4)) : (UNIFORM ? (TIMED ? 0 : 4) : 3);
}
template <int DH, bool UNIFORM, bool TIMED, bool JAGGED>
__global__ void __launch_bounds__(ATT_THREADS, JAGGED ? ext_jagged_min_blocks<DH, UNIFORM, TIMED>() : 0)
    hstu_attn_extend_kernel(HstuExtendArgs a) {
    pdl_wait();
    extern __shared__ __align__(16) unsigned char ext_smem_raw[];
    ExtSmem<DH>& sm = *reinterpret_cast<ExtSmem<DH>*>(ext_smem_raw);
    float* wcomb = reinterpret_cast<float*>(ext_smem_raw + sizeof(ExtSmem<DH>));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int qtiles = (a.n + ATT_BLK - 1) / ATT_BLK;
    const int h = blockIdx.y, b = blockIdx.z / qtiles, r0 = (blockIdx.z % qtiles) * ATT_BLK;
    const int k_lo = blockIdx.x * a.split;
    long long tok0 = 0;                                        // JAGGED: the sequence's first token row and its rows
    int rows = a.n;
    if constexpr (JAGGED) {
        seq_span(a.offsets, a.T, a.n, b, tok0, rows);
        if (r0 >= rows) return;                                // query tile past the end of a packed sequence
    }

    // positions of this thread's two rows (mma fragment rows g and g + 8 of the warp's 16)
    const int ra = r0 + warp * 16 + g, rb = ra + 8;
    const size_t row0 = JAGGED ? (size_t)tok0 : (size_t)b * a.n;
    const int pa = ra < rows ? a.pos[row0 + ra] : -1, pb = rb < rows ? a.pos[row0 + rb] : -1;
    if (tid == 0) sm.pmax = -1;
    // the partials' stores read the first row back from shared memory: no register holds it (or its address) across the key loop
    auto first_row = [&]() { return reinterpret_cast<long long*>(ext_smem_raw + sizeof(ExtSmem<DH>) + ext_table_bytes(a.bias.npos)); };
    if (JAGGED && tid == 0) *first_row() = tok0;
    __syncthreads();
    const int wmax = __reduce_max_sync(0xffffffffu, max(pa, pb));
    if (lane == 0) atomicMax(&sm.pmax, wmax);
    __syncthreads();
    const int pmax = sm.pmax;
    if (pmax < k_lo) return;                                   // no row of this tile reaches this split
    const int k_hi = min(k_lo + a.split, pmax + 1);            // keys [k_lo, k_hi)

    att_build_table(wcomb, a.bias, h, a.H, tid);
    if (TIMED)
        for (int i = tid; i <= ATT_MAX_BUCKETS; i += ATT_THREADS) sm.thr[i] = a.thr[i];
    const int u = a.users ? (int)a.users[b] : b;              // read only for a row that has a position: a valid user
    const bf16* gq = a.q + row0 * a.ldq + h * DH;
    const bf16* gk = a.kv + h * DH;
    const bf16* gv = gk + a.D;
    att_load_tile<DH>(sm.q, gq + (size_t)r0 * a.ldq, a.ldq, 0, 0, rows - r0, 0, tid);
    auto load_stream = [&](int k0, int buf) {                 // the tile's 64 keys lie in one page
        const size_t kr = a.pg.row(u, k0);
        att_load_tile<DH>(sm.kv[buf][0], gk + kr * 2 * a.D, 2 * a.D, 0, 0, k_hi - k0, 0, tid);
        att_load_tile<DH>(sm.kv[buf][1], gv + kr * 2 * a.D, 2 * a.D, 0, 0, k_hi - k0, 0, tid);
        if (TIMED && tid < ATT_BLK) sm.ts[buf][tid] = k0 + tid < k_hi ? a.ts[kr + tid] : 0;   // visible after the loop's barrier
    };
    load_stream(k_lo, 0);
    cp_async_commit();

    long long tqa = 0, tqb = 0;
    if (TIMED) {
        tqa = pa >= 0 ? a.ts[a.pg.row(u, pa)] : 0;
        tqb = pb >= 0 ? a.ts[a.pg.row(u, pb)] : 0;
    }
    const int warp_pmax = wmax;
    uint32_t qf[DH / 16][4];
    float o[DH / 8][4];
#pragma unroll
    for (int i = 0; i < DH / 8; ++i)
#pragma unroll
        for (int r = 0; r < 4; ++r) o[i][r] = 0.f;

    const int nt = (k_hi - k_lo + ATT_BLK - 1) / ATT_BLK;
    const unsigned masked = (unsigned)a.bias.npos * 64u;
    for (int it = 0; it < nt; ++it) {
        const int buf = it & 1, k0 = k_lo + it * ATT_BLK;
        if (it + 1 < nt) {
            load_stream(k0 + ATT_BLK, buf ^ 1);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (it == 0) att_load_afrag<DH>(qf, sm.q, warp * 16, lane);
        if (warp_pmax >= k0) {                                  // warp-uniform: some row of this warp sees a key of the tile
            float s[8][4];
            att_mma_nt<DH>(s, qf, sm.kv[buf][0], lane);
#pragma unroll
            for (int nb = 0; nb < 8; ++nb) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int hf = e >> 1, j = k0 + nb * 8 + 2 * t + (e & 1);
                    const int p = hf ? pb : pa;
                    unsigned ix = masked;
                    if (j <= p) {
                        ix = UNIFORM ? 0u : (unsigned)__ldg(a.pos_bucket + (p - j)) * 64u;
                        if (TIMED) ix += (unsigned)time_bucket_dev((hf ? tqb : tqa) - sm.ts[buf][j - k0], sm.thr, a.bias.ntime);
                    }
                    s[nb][e] = siluf(s[nb][e] + wcomb[ix]);
                }
            }
            uint32_t pf[4][4];
            att_pack_p(pf, s);
            att_mma_nn<DH>(o, pf, sm.kv[buf][1], lane);
        }
        __syncthreads();
    }

    // partial of this split for every row that reaches it (the combine reads splits 0 .. p / split of a row at position p)
    const size_t split0 = JAGGED ? (size_t)blockIdx.x * a.T : (size_t)blockIdx.x * a.B * a.n;   // the split's first partial row
    const size_t out0 = JAGGED ? (size_t)*first_row() : row0;
    float* dst = a.part + (split0 + out0) * a.D + h * DH;
#pragma unroll
    for (int i = 0; i < DH / 8; ++i) {
        const int col = i * 8 + 2 * t;
        if (pa >= k_lo) *reinterpret_cast<float2*>(dst + (size_t)ra * a.D + col) = make_float2(o[i][0], o[i][1]);
        if (pb >= k_lo) *reinterpret_cast<float2*>(dst + (size_t)rb * a.D + col) = make_float2(o[i][2], o[i][3]);
    }
}

// O[row, :] = bf16(sum over splits s = 0 .. pos[row] / split of part[s, row, :]) in split order ; 0 for rows without a position.
// One thread per 4 columns.
__global__ void __launch_bounds__(256) hstu_extend_combine_kernel(const float* __restrict__ part, const int* __restrict__ pos, int T, int D,
                                                                  int split, bf16* __restrict__ O) {
    pdl_wait();
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)T * D / 4) return;
    const int row = (int)(idx / (D / 4)), c = (int)(idx % (D / 4)) * 4;
    const int p = pos[row];
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p >= 0) {
        const int ns = p / split + 1;
        for (int s = 0; s < ns; ++s) {
            const float4 v = *reinterpret_cast<const float4*>(part + ((size_t)s * T + row) * D + c);
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
    }
    uint2 out;
    out.x = pack_bf16(acc.x, acc.y);
    out.y = pack_bf16(acc.z, acc.w);
    *reinterpret_cast<uint2*>(O + (size_t)row * D + c) = out;
}

// ---- page pool bookkeeping: one CTA per call, rows in order, so that which items find a page is a function of the call alone
constexpr int POOL_THREADS = 1024;
constexpr unsigned POOL_ERR_RANGE = 1u, POOL_ERR_REPEAT = 2u;   // bits of *errors

struct HstuPoolArgs {
    const long long* users; int B;     // [B] users of the call's rows
    const long long* ids; int n;       // [B, n] chunk ids (allocation only)
    int max_users, max_items, num_pages;
    int* page_table; int pt_ld, page_size;
    int* len; uint8_t* overflow;
    int* free_stack; int* free_top;    // free pages are free_stack[0 .. *free_top), the next one handed out is the top
    unsigned* errors;
    int* row_of;                       // [max_users] scratch: INT_MAX between calls
    int* room;                         // [B] out (allocation): items the row's user may now hold, -1 for a rejected row
    float* last_hidden; int ld_hidden; // [max_users, ld_hidden] rows zeroed on release (nullable)
};

// exclusive prefix sum of v over the CTA's POOL_THREADS threads; *total = the CTA's sum.  ws: 32 ints of shared memory
GRB_DEVINL int pool_scan(int v, int* ws, int* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) ws[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = ws[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        ws[lane] = w;
    }
    __syncthreads();
    const int before = warp ? ws[warp - 1] : 0;
    *total = ws[31];
    __syncthreads();
    return before + x - v;
}

// A row's user is accepted when it lies in [0, max_users) and no earlier row of the call names it; row_of[u] becomes the first
// row naming u.  Rejections set bits of *errors.
GRB_DEVINL void pool_mark_users(const HstuPoolArgs& a) {
    for (int b = threadIdx.x; b < a.B; b += POOL_THREADS) {
        const long long u = a.users[b];
        if (u >= 0 && u < a.max_users) atomicMin(&a.row_of[u], b);
        else atomicOr(a.errors, POOL_ERR_RANGE);
    }
    __syncthreads();
}
GRB_DEVINL int pool_user_of(const HstuPoolArgs& a, int b) {    // the row's user, or -1 for a rejected row
    const long long u = a.users[b];
    if (u < 0 || u >= a.max_users) return -1;
    if (*reinterpret_cast<volatile int*>(&a.row_of[u]) != b) {
        atomicOr(a.errors, POOL_ERR_REPEAT);
        return -1;
    }
    return (int)u;
}
GRB_DEVINL void pool_unmark_users(const HstuPoolArgs& a) {
    __syncthreads();
    for (int b = threadIdx.x; b < a.B; b += POOL_THREADS) {
        const long long u = a.users[b];
        if (u >= 0 && u < a.max_users) a.row_of[u] = 0x7fffffff;
    }
}

// Row b needs the pages that its user's items after this chunk (at most max_items) take beyond the ceil(len / page_size) the
// user holds.  Pages are popped from the top of the free stack in row order; a row that finds the stack empty gets what is left
// (possibly nothing) and its items beyond its pages are dropped by hstu_cache_append_kernel.  JAGGED: ids [T] of a packed chunk
// (a.n = max_len), and a row's valid items are counted over its sequence's token rows, seq_span(offsets, T, a.n, b).
template <bool JAGGED>
__global__ void __launch_bounds__(POOL_THREADS) hstu_pool_alloc_kernel(HstuPoolArgs a, const long long* __restrict__ offsets, int T) {
    pdl_wait();
    __shared__ int cnt[POOL_THREADS];
    __shared__ int ws[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int avail = *a.free_top;
    pool_mark_users(a);
    int handed = 0;                                            // pages asked for by the rows before this chunk
    for (int c0 = 0; c0 < a.B; c0 += POOL_THREADS) {
        const int rows = min(POOL_THREADS, a.B - c0);
        for (int r = warp; r < rows; r += 32) {                // valid items of each row: one warp per row
            int c = 0;
            if constexpr (JAGGED) {
                long long tok0;
                int len;
                seq_span(offsets, T, a.n, c0 + r, tok0, len);
                for (int j = lane; j < len; j += 32) c += a.ids[tok0 + j] != 0;
            } else {
                for (int j = lane; j < a.n; j += 32) c += a.ids[(size_t)(c0 + r) * a.n + j] != 0;
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
            if (lane == 0) cnt[r] = c;
        }
        __syncthreads();
        const int b = c0 + tid;
        int u = -1, have = 0, need = 0;
        if (tid < rows) {
            u = pool_user_of(a, b);
            if (u >= 0) {
                const int l = a.len[u];
                const int want = min(l + cnt[tid], a.max_items);
                have = (l + a.page_size - 1) / a.page_size;
                need = max(0, (want + a.page_size - 1) / a.page_size - have);
            }
        }
        int total;
        const int start = handed + pool_scan(need, ws, &total);
        const int got = max(0, min(need, avail - start));
        for (int k = 0; k < got; ++k) a.page_table[(size_t)u * a.pt_ld + have + k] = a.free_stack[avail - 1 - (start + k)];
        if (tid < rows) a.room[b] = u >= 0 ? min(a.max_items, (have + got) * a.page_size) : -1;
        handed += total;
        __syncthreads();                                       // cnt is rewritten by the next chunk
    }
    pool_unmark_users(a);
    if (tid == 0) *a.free_top = avail - min(handed, avail);
}

// Pushes each accepted row's pages back onto the free stack, in row order and then page order, and forgets the user: length,
// overflow flag and last hidden row become 0.
__global__ void __launch_bounds__(POOL_THREADS) hstu_pool_release_kernel(HstuPoolArgs a) {
    pdl_wait();
    __shared__ int ws[32];
    const int tid = threadIdx.x;
    const int top = *a.free_top;
    pool_mark_users(a);
    int pushed = 0;
    for (int c0 = 0; c0 < a.B; c0 += POOL_THREADS) {
        const int b = c0 + tid;
        const int u = b < a.B ? pool_user_of(a, b) : -1;
        const int pages = u >= 0 ? (a.len[u] + a.page_size - 1) / a.page_size : 0;
        int total;
        const int start = top + pushed + pool_scan(pages, ws, &total);
        for (int k = 0; k < pages; ++k)
            if (start + k < a.num_pages) a.free_stack[start + k] = a.page_table[(size_t)u * a.pt_ld + k];
        if (u >= 0) {
            a.len[u] = 0;
            a.overflow[u] = 0;
        }
        pushed += total;
    }
    if (a.last_hidden) {
        for (size_t i = tid; i < (size_t)a.B * a.ld_hidden; i += POOL_THREADS) {
            const long long u = a.users[i / a.ld_hidden];
            if (u >= 0 && u < a.max_users) a.last_hidden[(size_t)u * a.ld_hidden + i % a.ld_hidden] = 0.f;
        }
    }
    pool_unmark_users(a);
    if (tid == 0) *a.free_top = min(top + pushed, a.num_pages);
}

}  // namespace grb
