// genrec_b200 - HSTU attention: per-sequence timestamp pre-pass and the in-kernel time-bucket routine.
//
//   S[b,h,i,j] = Q_i . K_j + Wpos[pb0, h] + Wtime[tb(|ts_i - ts_j|), h]      valid = (j <= i) and not pad[b,j]
//
// The time bucket of an (i, j) cell can be derived from the two timestamps alone (integer thresholds that reproduce the
// reference's fp32 log/0.693 expression bit-exactly).  Per sequence a tiny pre-pass (hstu_seq_prep_kernel) rebases the int64
// timestamps to int32 offsets from the first valid event when the sequence spans < 2^31 ticks (always true for
// second-resolution data); sequences that do not fit take a 64-bit path.  hstu_bucket_bytes_debug_kernel exposes the routine
// cell by cell so that tests can pin it to the [B, L, L] bias-index matrix the attention kernels of attn_hstu.cuh read.
#pragma once
#include "attn_hstu.cuh"

namespace grb {

struct HstuBucketArgs {
    const long long* ts;        // [B, L] int64 or null (no temporal term)
    const int* rel32;           // [B, L] timestamp offsets (valid when wide[b] == 0)
    const uint8_t* wide;        // [B] 1: the sequence spans >= 2^31 ticks -> 64-bit bucket path
    const uint8_t* pad;         // [B, L] 1 = padded key
    const long long* thr64;     // [65] time-bucket thresholds (thr64[64] = INT64_MAX)
    int ntime;
    int B, L;
};

// ------------------------------------------------------------------------------------------------ per-sequence pre-pass
// rel[b, i] = int32(ts[b, i] - min_i ts[b, :]) ; wide[b] = 1 when max - min >= 2^31 (then rel is unused).  Padded positions take
// part: a padded QUERY row still attends to earlier real keys with its own timestamp (hstu.py:400 does not look at the pad mask), so
// with the usual "pads carry 0" convention the span is the largest real timestamp - fine for second-resolution data until 2038.
__global__ void __launch_bounds__(256) hstu_seq_prep_kernel(const long long* __restrict__ ts, const uint8_t* __restrict__ pad, int L,
                                                           int* __restrict__ rel, uint8_t* __restrict__ wide) {
    pdl_wait();
    (void)pad;
    __shared__ long long s_min[8], s_max[8];
    const int b = blockIdx.x;
    const long long* t = ts + (size_t)b * L;
    long long mn = 0x7fffffffffffffffLL, mx = -0x7fffffffffffffffLL - 1;
    for (int i = threadIdx.x; i < L; i += 256) { const long long v = t[i]; mn = v < mn ? v : mn; mx = v > mx ? v : mx; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const long long a = __shfl_xor_sync(0xffffffffu, mn, o), c = __shfl_xor_sync(0xffffffffu, mx, o);
        mn = a < mn ? a : mn; mx = c > mx ? c : mx;
    }
    if ((threadIdx.x & 31) == 0) { s_min[threadIdx.x >> 5] = mn; s_max[threadIdx.x >> 5] = mx; }
    __syncthreads();
    mn = s_min[0]; mx = s_max[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) { mn = s_min[w] < mn ? s_min[w] : mn; mx = s_max[w] > mx ? s_max[w] : mx; }
    // span computed in unsigned arithmetic: mx - mn of two int64 may not fit int64
    const unsigned long long span = (unsigned long long)mx - (unsigned long long)mn;
    const bool w64 = span >= (1ull << 31);
    if (threadIdx.x == 0) wide[b] = w64 ? 1 : 0;
    for (int i = threadIdx.x; i < L; i += 256) rel[(size_t)b * L + i] = w64 ? 0 : (int)(t[i] - mn);
}

// ------------------------------------------------------------------------------------------------ bucket bytes of 32 cells
// cells (row i, keys j0 .. j0+31) ; bk[k >> 2] byte (k & 3) = time bucket of cell k, or 64 when the cell is masked.
// s_rel / s_ts / s_pad point at the first of the 32 keys in shared memory.
struct AtcBk8 {
    uint32_t w[8];
};
// 32-bit path (the sequence spans < 2^31 ticks): inlined, this is the hot one
template <bool MASKED>
GRB_DEVINL void atc_buckets_narrow(uint32_t (&bk)[8], int i, int j0, int ri, const int* s_rel, const uint8_t* s_pad, const uint32_t* s_thr32,
                                   int ntime, int L, bool row_ok) {
    const int ntm1 = ntime - 1;
    const bool clamp = ntm1 < 31;     // 32-bit differences never reach bucket 32 (warp-uniform)
#pragma unroll
    for (int w = 0; w < 8; ++w) {
        uint32_t word = 0;
        const int4 r4 = *reinterpret_cast<const int4*>(s_rel + 4 * w);      // four keys per broadcast LDS.128
        const int rj[4] = {r4.x, r4.y, r4.z, r4.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int k = w * 4 + q;
            int b = 0;
            if (ntime > 0) {
                // e = floor(log2 |d|) (-1 for d == 0: thr32[0] == 0 then gives bucket 0) ; bucket = e + (|d| >= thr[e + 1])
                const int d = ri - rj[q];
                const unsigned a = (unsigned)(d < 0 ? -d : d);
                const int e = 31 - __clz(a);
                b = e + (a >= s_thr32[e + 1] ? 1 : 0);
                if (clamp) b = b < ntm1 ? b : ntm1;
            }
            if (MASKED) {
                const int j = j0 + k;
                const bool valid = row_ok && j <= i && j < L && s_pad[k] == 0;
                b = valid ? b : 64;
            }
            word |= (uint32_t)b << (8 * q);
        }
        bk[w] = word;
    }
}
// 64-bit path: a sequence that spans >= 2^31 ticks (millisecond clocks, synthetic extremes).  Out of line on purpose: it is
// rare and its 64-bit arithmetic would otherwise be inlined at every call site (instruction-cache footprint of the hot loop).
// g_ts points at the timestamps of the 32 keys in GLOBAL memory.
__device__ __noinline__ AtcBk8 atc_buckets_wide(int i, int j0, long long ti, const long long* g_ts, const uint8_t* s_pad,
                                                const long long* thr64, int ntime, int L, int row_ok) {
    AtcBk8 out;
    for (int w = 0; w < 8; ++w) {
        uint32_t word = 0;
        for (int q = 0; q < 4; ++q) {
            const int k = w * 4 + q;
            const int j = j0 + k;
            int b = 0;
            if (ntime > 0 && j < L) b = time_bucket_dev(ti - g_ts[k], thr64, ntime);
            const bool valid = row_ok && j <= i && j < L && s_pad[k] == 0;
            b = valid ? b : 64;
            word |= (uint32_t)b << (8 * q);
        }
        out.w[w] = word;
    }
    return out;
}
// bucket bytes of one (row, 32-key chunk): classification -> all masked / narrow fast / narrow masked / wide
GRB_DEVINL bool atc_chunk_buckets(uint32_t (&bk)[8], int q_first, int lane, int i, int j0, int ri, long long ti, bool wide, const int* s_rel,
                                  const long long* g_ts, const uint8_t* s_pad, const uint32_t* s_thr32, const long long* thr64, int ntime, int L,
                                  bool row_ok);
GRB_DEVINL void atc_buckets_all_masked(uint32_t (&bk)[8]) {
#pragma unroll
    for (int w = 0; w < 8; ++w) bk[w] = 0x40404040u;
}

// classification of a (32-row block, 32-key chunk) pair, warp-uniform
struct AtcChunkClass {
    bool all_masked, needs_mask;
};
GRB_DEVINL AtcChunkClass atc_classify(int q_first, int k_first, int L, const uint8_t* s_pad_chunk, int lane) {
    AtcChunkClass cc;
    cc.all_masked = q_first >= L || k_first >= L || k_first > q_first + 31;
    const bool any_pad = __any_sync(0xffffffffu, s_pad_chunk[lane] != 0);
    cc.needs_mask = any_pad || (k_first + 31 > q_first) || (q_first + 31 >= L) || (k_first + 31 >= L);
    return cc;
}

GRB_DEVINL bool atc_chunk_buckets(uint32_t (&bk)[8], int q_first, int lane, int i, int j0, int ri, long long ti, bool wide, const int* s_rel,
                                  const long long* g_ts, const uint8_t* s_pad, const uint32_t* s_thr32, const long long* thr64, int ntime, int L,
                                  bool row_ok) {
    const AtcChunkClass cl = atc_classify(q_first, j0, L, s_pad, lane);
    if (cl.all_masked) {
        atc_buckets_all_masked(bk);
    } else if (wide) {
        const AtcBk8 r = atc_buckets_wide(i, j0, ti, g_ts, s_pad, thr64, ntime, L, row_ok ? 1 : 0);
#pragma unroll
        for (int w = 0; w < 8; ++w) bk[w] = r.w[w];
    } else if (cl.needs_mask) {
        atc_buckets_narrow<true>(bk, i, j0, ri, s_rel, s_pad, s_thr32, ntime, L, row_ok);
    } else {
        atc_buckets_narrow<false>(bk, i, j0, ri, s_rel, s_pad, s_thr32, ntime, L, row_ok);
    }
    return cl.all_masked;
}

// Test hook: the bucket / mask byte of every (i, j) cell, produced by the routine the attention kernels use (same
// classification, same fast / masked / wide variants).  grid (ceil(L / 32), ceil(L / 128), B), block 128.
__global__ void __launch_bounds__(128) hstu_bucket_bytes_debug_kernel(HstuBucketArgs a, uint8_t* __restrict__ out) {
    pdl_wait();
    __shared__ __align__(16) int s_rel[32];
    __shared__ uint8_t s_pad[32];
    __shared__ uint32_t s_thr32[36];
    const int b = blockIdx.z, q0 = blockIdx.y * 128, j0 = blockIdx.x * 32;
    const int L = a.L, t = threadIdx.x, sub = t >> 5, lane = t & 31;
    const long long tok0 = (long long)b * L;
    const bool has_time = a.ts != nullptr && a.ntime > 0;
    const int ntime = has_time ? a.ntime : 0;
    const bool wide = has_time && a.wide[b] != 0;
    for (int k = t; k < 36; k += 128) s_thr32[k] = k <= 31 ? (uint32_t)a.thr64[k] : 0xffffffffu;
    if (t < 32) {
        const int j = j0 + t;
        int kr = 0; uint8_t kp = 1;
        if (j < L) {
            kp = a.pad[tok0 + j];
            if (has_time && !wide) kr = a.rel32[tok0 + j];
        }
        s_rel[t] = kr; s_pad[t] = kp;
    }
    __syncthreads();
    const int i = q0 + t;
    const bool row_ok = i < L;
    const int ri = (has_time && !wide && row_ok) ? a.rel32[tok0 + i] : 0;
    const long long ti = (wide && row_ok) ? a.ts[tok0 + i] : 0;
    uint32_t bk[8];
    atc_chunk_buckets(bk, q0 + sub * 32, lane, i, j0, ri, ti, wide, s_rel, a.ts != nullptr ? a.ts + tok0 + j0 : nullptr, s_pad, s_thr32, a.thr64,
                      ntime, L, row_ok);
    if (row_ok)
        for (int k = 0; k < 32; ++k)
            if (j0 + k < L) out[(size_t)(tok0 + i) * L + j0 + k] = (uint8_t)((bk[k >> 2] >> (8 * (k & 3))) & 0xffu);
}

}  // namespace grb
