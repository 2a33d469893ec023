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
#pragma once
#include "attn_hstu.cuh"

namespace grb {

// One warp per user.  pos[b, r] = len[b] + (valid rows of the chunk before r) for a valid row (id != 0), -1 for a pad
// and for an item that does not fit in `cap` (dropped; overflow[b] = 1).  The chunk's timestamps are written into the
// cache, len[b] becomes min(len[b] + valid, cap) and last_row[b] is the chunk row of the user's last valid item, or -1.
__global__ void __launch_bounds__(128) hstu_cache_append_kernel(const long long* __restrict__ ids, const long long* __restrict__ ts, int B,
                                                                int n, int cap, long long* __restrict__ cache_ts, int* __restrict__ len,
                                                                uint8_t* __restrict__ overflow, int* __restrict__ pos,
                                                                int* __restrict__ last_row) {
    pdl_wait();
    const int b = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (b >= B) return;
    const int base = len[b];
    int count = 0, last = -1;
    for (int r0 = 0; r0 < n; r0 += 32) {
        const int r = r0 + lane;
        const bool valid = r < n && ids[(size_t)b * n + r] != 0;
        const unsigned m = __ballot_sync(0xffffffffu, valid);
        const int q = base + count + __popc(m & ((1u << lane) - 1u));
        if (r < n) {
            int p = -1;
            if (valid && q < cap) {
                p = q;
                cache_ts[(size_t)b * cap + q] = ts ? ts[(size_t)b * n + r] : 0;
            }
            pos[(size_t)b * n + r] = p;
        }
        if (m) last = r0 + 31 - __clz((int)m);
        count += __popc(m);
    }
    if (lane == 0) {
        const long long total = (long long)base + count;
        len[b] = total > cap ? cap : (int)total;
        if (total > cap) overflow[b] = 1;
        last_row[b] = last;
    }
}

// kv[b, pos, 0:D) = K row, kv[b, pos, D:2D) = V row of every chunk row with pos >= 0.  P = [U | V | Q | K] [B*n, 4D] bf16.
// One thread per 16-byte piece.
__global__ void __launch_bounds__(256) hstu_kv_scatter_kernel(const bf16* __restrict__ P, const int* __restrict__ pos, int T, int n, int D,
                                                              int cap, bf16* __restrict__ kv) {
    pdl_wait();
    const int per_row = 2 * D / 8;
    const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= (size_t)T * per_row) return;
    const int row = (int)(idx / per_row), c = (int)(idx % per_row) * 8;   // column of the cache row
    const int p = pos[row];
    if (p < 0) return;
    const int b = row / n;
    const int src = c < D ? 3 * D + c : c;                                // K = P[:, 3D:4D) ; V = P[:, D:2D)
    *reinterpret_cast<uint4*>(kv + ((size_t)b * cap + p) * 2 * D + c) =
        *reinterpret_cast<const uint4*>(P + (size_t)row * 4 * D + src);
}

struct HstuExtendArgs {
    const bf16* q; int ldq;            // chunk queries, [B * n] rows (P + 2D, ld 4D)
    const bf16* kv;                    // this layer's cache [B, cap, 2D]: K | V
    const long long* ts;               // [B, cap] cache timestamps
    const int* pos;                    // [B * n] cache position of each chunk row, -1 = none
    const uint8_t* pos_bucket;         // [cap] bucket of delta = p_i - j ; null: every delta uses the single live row of bias.wpos
    const long long* thr;              // [65] time-bucket thresholds
    HstuBiasArgs bias;                 // wpos / wtime / npos / ntime (bias_index unused)
    int B, n, H, D, cap;
    int split;                         // keys per CTA, a multiple of ATT_BLK ; grid.x = ceil(cap / split)
    float* part;                       // [grid.x, B * n, D] fp32 partial outputs
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
// dynamic tail: float wcomb[npos * 64 + 1] (att_build_table)

// grid (ceil(cap / split), H, B * ceil(n / 64)), 128 threads: 64 chunk rows of one user and head against the keys
// [split * x, split * (x + 1)) of the user's cache.  Tiles that lie beyond every row's position are skipped.
template <int DH, bool UNIFORM, bool TIMED>
__global__ void __launch_bounds__(ATT_THREADS) hstu_attn_extend_kernel(HstuExtendArgs a) {
    pdl_wait();
    extern __shared__ __align__(16) unsigned char ext_smem_raw[];
    ExtSmem<DH>& sm = *reinterpret_cast<ExtSmem<DH>*>(ext_smem_raw);
    float* wcomb = reinterpret_cast<float*>(ext_smem_raw + sizeof(ExtSmem<DH>));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, t = lane & 3;
    const int qtiles = (a.n + ATT_BLK - 1) / ATT_BLK;
    const int h = blockIdx.y, b = blockIdx.z / qtiles, r0 = (blockIdx.z % qtiles) * ATT_BLK;
    const int k_lo = blockIdx.x * a.split;

    // positions of this thread's two rows (mma fragment rows g and g + 8 of the warp's 16)
    const int ra = r0 + warp * 16 + g, rb = ra + 8;
    const size_t row0 = (size_t)b * a.n;
    const int pa = ra < a.n ? a.pos[row0 + ra] : -1, pb = rb < a.n ? a.pos[row0 + rb] : -1;
    if (tid == 0) sm.pmax = -1;
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
    const bf16* gq = a.q + row0 * a.ldq + h * DH;
    const bf16* gk = a.kv + (size_t)b * a.cap * 2 * a.D + h * DH;
    const bf16* gv = gk + a.D;
    const long long* gts = a.ts + (size_t)b * a.cap;
    att_load_tile<DH>(sm.q, gq + (size_t)r0 * a.ldq, a.ldq, 0, 0, a.n - r0, 0, tid);
    auto load_stream = [&](int k0, int buf) {
        att_load_tile<DH>(sm.kv[buf][0], gk + (size_t)k0 * 2 * a.D, 2 * a.D, 0, 0, k_hi - k0, 0, tid);
        att_load_tile<DH>(sm.kv[buf][1], gv + (size_t)k0 * 2 * a.D, 2 * a.D, 0, 0, k_hi - k0, 0, tid);
        if (TIMED && tid < ATT_BLK) sm.ts[buf][tid] = k0 + tid < k_hi ? gts[k0 + tid] : 0;   // visible after the loop's barrier
    };
    load_stream(k_lo, 0);
    cp_async_commit();

    long long tqa = 0, tqb = 0;
    if (TIMED) {
        tqa = pa >= 0 ? gts[pa] : 0;
        tqb = pb >= 0 ? gts[pb] : 0;
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
    float* dst = a.part + ((size_t)blockIdx.x * a.B * a.n + row0) * a.D + h * DH;
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

}  // namespace grb
