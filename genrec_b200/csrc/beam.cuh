// genrec_b200 - trie-constrained beam step of TIGER's generate() on the device (genrec/models/tiger.py:312-452).
//
// The reference masks the logits with a Python double loop over (batch, beam) walking a dict trie, and picks the next beams with a
// per-batch Python loop calling .item() on every candidate: the decode is host-bound.  Here the trie is a CSR over node ids
// (child_off [n_nodes + 1], child_tok / child_node [n_edges], children sorted by token, root = node 0, dead = -1) and a decode step is
// two launches:
//   trie_log_softmax_kernel   legal-token mask from the node's children (or the step's vocabulary range without a trie),
//                             masked_fill(-1e32) / temperature, softmax AND log_softmax                 (tiger.py:364-384)
//   beam_select_kernel        total = beam_logp + cand_logp, descending sort, first K candidates whose token sequence is new,
//                             -1e32 / zero-sequence / root-node fillers, trie descent of the survivors   (tiger.py:386-441)
//                             (K <= 32, K * KK <= 1024; wider steps: the four launches of the wide beam step below)
// Candidate sampling stays torch.multinomial on the probabilities produced here (the reference's RNG stream is part of its output).
#pragma once
#include "common.cuh"
#include "tc_gemm.cuh"   // exp_accurate

namespace grb {

struct TrieCsr {
    const int* child_off;    // [n_nodes + 1]
    const int* child_tok;    // [n_edges] raw token ids (0 .. num_embeddings-1), ascending inside a node
    const int* child_node;   // [n_edges]
    int n_nodes;
};

// one CTA per beam row.  node < 0 (dead) or a leaf: no legal token -> every entry is -1e32 / T, i.e. the uniform distribution, exactly
// as the reference's masked_fill produces it.  use_trie = 0: legal = [vocab_offset, vocab_offset + num_emb), the rest is -inf.
__global__ void __launch_bounds__(256) trie_log_softmax_kernel(const float* __restrict__ logits, int V, const int* __restrict__ node,
                                                               TrieCsr trie, int use_trie, int vocab_offset, int num_emb, float temperature,
                                                               float* __restrict__ probs, float* __restrict__ logp) {
    pdl_wait();
    extern __shared__ unsigned beam_smem[];
    unsigned* legal = beam_smem;                       // bitmap, ceil(V / 32) words
    __shared__ float red[8];
    __shared__ float bc[2];
    const int row = blockIdx.x, tid = threadIdx.x;
    const int words = (V + 31) >> 5;
    for (int w = tid; w < words; w += 256) legal[w] = 0u;
    __syncthreads();
    if (use_trie) {
        const int nd = node[row];
        if (nd >= 0 && nd < trie.n_nodes) {
            const int c0 = trie.child_off[nd], c1 = trie.child_off[nd + 1];
            for (int c = c0 + tid; c < c1; c += 256) {
                const int v = vocab_offset + trie.child_tok[c];
                if (v >= 0 && v < V) atomicOr(&legal[v >> 5], 1u << (v & 31));
            }
        }
    } else {
        for (int v = vocab_offset + tid; v < vocab_offset + num_emb && v < V; v += 256)
            if (v >= 0) atomicOr(&legal[v >> 5], 1u << (v & 31));
    }
    __syncthreads();
    const float* x = logits + (size_t)row * V;
    const float fill = use_trie ? -1e32f : -INFINITY;
    // logits / temperature exactly as the reference rounds it (a true division, and no contraction of the later "- max" into an FMA:
    // a dead node's row is -1e32 / T everywhere and must come out as EXACTLY equal entries, i.e. the uniform distribution)
    auto val = [&](int v) { return __fdiv_rn(((legal[v >> 5] >> (v & 31)) & 1u) ? x[v] : fill, temperature); };
    float m = -INFINITY;
    for (int v = tid; v < V; v += 256) m = fmaxf(m, val(v));
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) red[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) { float t = red[0]; for (int w = 1; w < 8; ++w) t = fmaxf(t, red[w]); bc[0] = t; }
    __syncthreads();
    m = bc[0];
    float s = 0.f;
    for (int v = tid; v < V; v += 256) s += exp_accurate(__fsub_rn(val(v), m));
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    __syncthreads();
    if ((tid & 31) == 0) red[tid >> 5] = s;
    __syncthreads();
    if (tid == 0) { float t = 0.f; for (int w = 0; w < 8; ++w) t += red[w]; bc[1] = t; }
    __syncthreads();
    const float sum = bc[1];
    const float lsum = 0.6931471805599453f * __log2f(sum);
    for (int v = tid; v < V; v += 256) {
        const float d = __fsub_rn(val(v), m);
        probs[(size_t)row * V + v] = __fdiv_rn(exp_accurate(d), sum);
        logp[(size_t)row * V + v] = d - lsum;
    }
}

struct BeamSelectArgs {
    const long long* beam_seqs;   // [B, K, S]
    const float* beam_logps;      // [B, K]
    const long long* cand_tok;    // [B, K, KK]  raw token ids (vocabulary index - vocab_offset)
    const float* cand_logp;       // [B, K, KK]
    const int* nodes;             // [B, K] (nullable: no trie)
    TrieCsr trie;
    int K, KK, S;
    long long* new_seqs;          // [B, K, S + 1]
    float* new_logps;             // [B, K]
    int* new_nodes;               // [B, K] (nullable)
};
constexpr int BEAM_MAX_CAND = 1024;

// beam k of row b continues parent p with token t: the parent's sequence + t, its total, and the trie node it reaches
GRB_DEVINL void beam_emit(const BeamSelectArgs& a, int b, int k, int p, long long t, float total) {
    long long* out = a.new_seqs + ((size_t)b * a.K + k) * (a.S + 1);
    const long long* seq = a.beam_seqs + ((size_t)b * a.K + p) * a.S;
    for (int s = 0; s < a.S; ++s) out[s] = seq[s];
    out[a.S] = t;
    a.new_logps[(size_t)b * a.K + k] = total;
    if (a.new_nodes) {
        int nd = a.nodes ? a.nodes[(size_t)b * a.K + p] : -1, child = -1;
        if (nd >= 0 && nd < a.trie.n_nodes) {
            int lo = a.trie.child_off[nd], hi = a.trie.child_off[nd + 1];
            while (lo < hi) {                       // children are sorted by token
                const int mid = (lo + hi) >> 1;
                const int tk = a.trie.child_tok[mid];
                if (tk == t) { child = a.trie.child_node[mid]; break; }
                if (tk < t) lo = mid + 1; else hi = mid;
            }
        }
        a.new_nodes[(size_t)b * a.K + k] = child;   // parent_node.get(tid, DEAD_NODE)            (tiger.py:419-421)
    }
}
// fewer than K distinct candidates: the zero sequence, -1e32 and the root                             (tiger.py:423-429)
GRB_DEVINL void beam_fill(const BeamSelectArgs& a, int b, int k) {
    long long* out = a.new_seqs + ((size_t)b * a.K + k) * (a.S + 1);
    for (int s = 0; s <= a.S; ++s) out[s] = 0;
    a.new_logps[(size_t)b * a.K + k] = -1e32f;
    if (a.new_nodes) a.new_nodes[(size_t)b * a.K + k] = 0;
}

// one CTA (1024 threads) per batch row; K <= 32, K * KK <= 1024.  Order of equal totals: lower flat candidate index first.
__global__ void __launch_bounds__(BEAM_MAX_CAND) beam_select_kernel(BeamSelectArgs a) {
    pdl_wait();
    __shared__ float s_key[BEAM_MAX_CAND];
    __shared__ int s_idx[BEAM_MAX_CAND];
    __shared__ int s_cls[32];
    __shared__ int s_pick[32];
    __shared__ int s_npick;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = a.K * a.KK;
    const long long* seqs = a.beam_seqs + (size_t)b * a.K * a.S;
    // parents whose token sequences are identical produce identical children: class = the smallest such parent
    if (tid < a.K) {
        int c = tid;
        for (int p = 0; p < tid; ++p) {
            bool same = true;
            for (int t = 0; t < a.S; ++t) same = same && seqs[(size_t)p * a.S + t] == seqs[(size_t)tid * a.S + t];
            if (same) { c = p; break; }
        }
        s_cls[tid] = c;
    }
    if (tid < n) {
        const int p = tid / a.KK;
        s_key[tid] = a.beam_logps[(size_t)b * a.K + p] + a.cand_logp[(size_t)b * n + tid];    // (tiger.py:393)
        s_idx[tid] = tid;
    } else {
        s_key[tid] = -INFINITY;
        s_idx[tid] = 0x7fffffff;
    }
    __syncthreads();
    // bitonic sort, descending by key, ascending by index among equal keys (NaN never occurs: log-probabilities)
    for (int k = 2; k <= BEAM_MAX_CAND; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            const int o = tid ^ j;
            if (o > tid) {
                const float ka = s_key[tid], kb = s_key[o];
                const int ia = s_idx[tid], ib = s_idx[o];
                const bool a_first = ka > kb || (ka == kb && ia < ib);   // a belongs before b in the final order
                const bool up = (tid & k) == 0;
                if (up ? !a_first : a_first) { s_key[tid] = kb; s_key[o] = ka; s_idx[tid] = ib; s_idx[o] = ia; }
            }
            __syncthreads();
        }
    }
    // greedy scan by one warp: lane l remembers the l-th pick
    if (tid < 32) {
        int my_cls = -1; long long my_tok = -1;
        int npick = 0;
        for (int j = 0; j < n && npick < a.K; ++j) {
            const int ci = s_idx[j];
            const int p = ci / a.KK;
            const long long t = a.cand_tok[(size_t)b * n + ci];
            const int c = s_cls[p];
            const bool dup = tid < npick && my_cls == c && my_tok == t;
            if (__ballot_sync(0xffffffffu, dup) == 0u) {
                if (tid == npick) { my_cls = c; my_tok = t; s_pick[npick] = j; }
                ++npick;
            }
        }
        if (tid == 0) s_npick = npick;
    }
    __syncthreads();
    const int npick = s_npick;
    if (tid < a.K) {
        if (tid < npick) {
            const int ci = s_idx[s_pick[tid]];
            beam_emit(a, b, tid, ci / a.KK, a.cand_tok[(size_t)b * n + ci], s_key[s_pick[tid]]);
        } else {
            beam_fill(a, b, tid);
        }
    }
}

// ------------------------------------------------------------------------------------------------ wide beam step
// The same contract for 1 <= K <= 1024, K * KK <= 262,144 candidates per row.  A candidate is picked iff it is the first occurrence
// of its (parent class, token) in the order AND fewer than K first occurrences precede it, so the greedy scan becomes three
// data-parallel passes and a per-row selection:
//   beam_class_kernel         class of every parent = the smallest parent with the same token sequence           (one CTA per row)
//   beam_dedup_insert_kernel  hash table per row: (class, token) -> the largest key among its candidates        (grid-stride)
//   beam_dedup_mark_kernel    mono[i] = the monotone total of candidate i if it holds its group's slot, else 0    (grid-stride)
//   beam_wide_select_kernel   beam_radix_topk (radix select of the K-th largest mono, index-ordered ties, a sort of the K picks;
//                             COBRA's beam step shares it), then the output of beam_emit / beam_fill            (one CTA per row)
// key = monotone total << 32 | (2^32 - 1 - flat index): unique per candidate, larger = earlier in the order; 0 never occurs (the
// flat index is < 2^18), so 0 marks an empty slot.  The selected set and its order do not depend on which CTA inserts first.
constexpr int BEAM_WIDE_MAX_K = 1024;
constexpr int BEAM_WIDE_MAX_CAND = 262144;
constexpr int BEAM_WIDE_THREADS = 1024;

struct BeamWideArgs {
    BeamSelectArgs s;
    int B;
    int cap_log2;                   // hash slots per row = 2^cap_log2 >= 2 K KK
    int* cls;                       // [B, K]
    unsigned long long* table;      // [B, 2^cap_log2], zeroed
    unsigned* mono;                 // [B, K KK]
};

// order-preserving map of a total onto unsigned (-0 and +0 are one value, as in the reference's sort); -inf -> 0x007fffff > 0
GRB_DEVINL unsigned beam_mono(float f) {
    const unsigned u = __float_as_uint(f == 0.f ? 0.f : f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
GRB_DEVINL unsigned long long beam_key(unsigned mono, int flat) {
    return ((unsigned long long)mono << 32) | (0xffffffffu - (unsigned)flat);
}
GRB_DEVINL int beam_key_flat(unsigned long long key) { return (int)(0xffffffffu - (unsigned)key); }
GRB_DEVINL size_t beam_slot(int cls, long long tok, int cap_log2) {
    unsigned long long h = (unsigned long long)tok * 0x9e3779b97f4a7c15ull ^ ((unsigned long long)cls << 32 | (unsigned)cls);
    h ^= h >> 31; h *= 0xbf58476d1ce4e5b9ull; h ^= h >> 29;
    return (size_t)(h >> (64 - cap_log2));
}

__global__ void __launch_bounds__(BEAM_WIDE_THREADS) beam_class_kernel(BeamWideArgs w) {
    pdl_wait();
    __shared__ unsigned long long s_hash[BEAM_WIDE_MAX_K];
    const BeamSelectArgs& a = w.s;
    const int b = blockIdx.x, tid = threadIdx.x;
    const long long* seqs = a.beam_seqs + (size_t)b * a.K * a.S;
    for (int p = tid; p < a.K; p += BEAM_WIDE_THREADS) {             // a fingerprint first, the sequences only where it matches
        unsigned long long h = 0;
        for (int t = 0; t < a.S; ++t) h = (h ^ (unsigned long long)seqs[(size_t)p * a.S + t]) * 0x100000001b3ull + 0x9e3779b97f4a7c15ull;
        s_hash[p] = h;
    }
    __syncthreads();
    for (int p = tid; p < a.K; p += BEAM_WIDE_THREADS) {
        int c = p;
        for (int q = 0; q < p; ++q) {
            if (s_hash[q] != s_hash[p]) continue;
            bool same = true;
            for (int t = 0; t < a.S && same; ++t) same = seqs[(size_t)q * a.S + t] == seqs[(size_t)p * a.S + t];
            if (same) { c = q; break; }
        }
        w.cls[(size_t)b * a.K + p] = c;
    }
}

__global__ void __launch_bounds__(256) beam_dedup_insert_kernel(BeamWideArgs w) {
    pdl_wait();
    const BeamSelectArgs& a = w.s;
    const size_t n = (size_t)a.K * a.KK, total = (size_t)w.B * n, mask = ((size_t)1 << w.cap_log2) - 1;
    for (size_t e = (size_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (size_t)gridDim.x * 256) {
        const size_t b = e / n;
        const int f = (int)(e - b * n), p = f / a.KK;
        const int c = w.cls[b * a.K + p];
        const long long t = a.cand_tok[e];
        const unsigned long long key = beam_key(beam_mono(a.beam_logps[b * a.K + p] + a.cand_logp[e]), f);
        unsigned long long* tab = w.table + (b << w.cap_log2);
        for (size_t h = beam_slot(c, t, w.cap_log2);; h = (h + 1) & mask) {
            const unsigned long long v = atomicCAS(&tab[h], 0ull, key);
            if (v == 0ull) break;
            // the slot's (class, token) is that of any key it ever held: atomicMax only ever stores keys of the same group
            const int fo = beam_key_flat(v);
            if (w.cls[b * a.K + fo / a.KK] == c && a.cand_tok[b * n + fo] == t) { atomicMax(&tab[h], key); break; }
        }
    }
}

__global__ void __launch_bounds__(256) beam_dedup_mark_kernel(BeamWideArgs w) {
    pdl_wait();
    const BeamSelectArgs& a = w.s;
    const size_t n = (size_t)a.K * a.KK, total = (size_t)w.B * n, mask = ((size_t)1 << w.cap_log2) - 1;
    for (size_t e = (size_t)blockIdx.x * 256 + threadIdx.x; e < total; e += (size_t)gridDim.x * 256) {
        const size_t b = e / n;
        const int f = (int)(e - b * n), p = f / a.KK;
        const int c = w.cls[b * a.K + p];
        const long long t = a.cand_tok[e];
        const unsigned m = beam_mono(a.beam_logps[b * a.K + p] + a.cand_logp[e]);
        const unsigned long long key = beam_key(m, f);
        const unsigned long long* tab = w.table + (b << w.cap_log2);
        unsigned long long v;
        for (size_t h = beam_slot(c, t, w.cap_log2);; h = (h + 1) & mask) {
            v = tab[h];
            if (v == key) break;
            const int fo = beam_key_flat(v);
            if (w.cls[b * a.K + fo / a.KK] == c && a.cand_tok[b * n + fo] == t) break;
        }
        w.mono[e] = v == key ? m : 0u;
    }
}

// Shared memory of beam_radix_topk.
struct BeamRadixSmem {
    unsigned hist[256];
    unsigned long long key[BEAM_WIDE_MAX_K];
    int warp[BEAM_WIDE_THREADS / 32];
    unsigned prefix;
    int need, cnt, all;
};

// The K largest nonzero entries of mono [n] (n < 2^31), by all BEAM_WIDE_THREADS threads of the CTA: radix select of the K-th
// largest value, index-ordered ties, then a sort of the picks.  Returns the number of picks (min(K, nonzero entries)); s.key[0 ..]
// holds their beam_key, largest first (equal values: the lower index first).
GRB_DEVINL int beam_radix_topk(const unsigned* mono, int n, int K, BeamRadixSmem& s) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) { s.prefix = 0u; s.need = K; s.cnt = 0; s.all = 0; }
    // radix select, 8 bits at a time from the top, of the K-th largest nonzero mono (the threshold T = s.prefix); s.need ends as
    // the number of entries equal to T that are picked.  With at most K nonzero entries, every one is picked.
    unsigned pmask = 0u;
    for (int shift = 24; shift >= 0; shift -= 8) {
        if (tid < 256) s.hist[tid] = 0u;
        __syncthreads();
        const unsigned prefix = s.prefix;
        for (int i = tid; i < n; i += BEAM_WIDE_THREADS) {
            const unsigned v = mono[i];
            if (v != 0u && (v & pmask) == prefix) atomicAdd(&s.hist[(v >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (warp == 0) {                                  // lane l holds bins 255 - 8 l ... 248 - 8 l, largest digit first
            unsigned c[8], sum = 0u;
#pragma unroll
            for (int j = 0; j < 8; ++j) { c[j] = s.hist[255 - 8 * lane - j]; sum += c[j]; }
            unsigned incl = sum;
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned u = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += u;
            }
            const unsigned need = (unsigned)s.need;
            const unsigned all = __shfl_sync(0xffffffffu, incl, 31);
            if (shift == 24 && all <= need) {
                if (lane == 0) s.all = 1;
            } else {
                const unsigned hit = __ballot_sync(0xffffffffu, incl >= need);
                if (lane == __ffs(hit) - 1) {
                    unsigned above = incl - sum;
                    int j = 0;
                    while (above + c[j] < need) above += c[j++];
                    s.prefix = prefix | ((unsigned)(255 - 8 * lane - j) << shift);
                    s.need = (int)(need - above);
                }
            }
        }
        __syncthreads();
        if (s.all) break;
        pmask |= 255u << shift;
    }
    const bool all = s.all != 0;
    const unsigned T = all ? 0u : s.prefix;
    const int need = all ? 0 : s.need;
    // collect the picks: every entry above T, and the `need` ones equal to T with the lowest index
    int tie_base = 0;
    for (int base = 0; base < n; base += BEAM_WIDE_THREADS) {
        const int i = base + tid;
        const unsigned v = i < n ? mono[i] : 0u;
        const bool tie = need > 0 && v == T;
        const unsigned bal = __ballot_sync(0xffffffffu, tie);
        if (lane == 0) s.warp[warp] = __popc(bal);
        __syncthreads();
        int rank = tie_base + __popc(bal & ((1u << lane) - 1u)), tile = 0;
        for (int q = 0; q < BEAM_WIDE_THREADS / 32; ++q) {
            const int cq = s.warp[q];
            if (q < warp) rank += cq;
            tile += cq;
        }
        if (v > T || (tie && rank < need)) s.key[atomicAdd(&s.cnt, 1)] = beam_key(v, i);
        tie_base += tile;
        __syncthreads();
    }
    const int npick = s.cnt;
    int P = 1;
    while (P < K) P <<= 1;
    if (tid < P && tid >= npick) s.key[tid] = 0ull;
    __syncthreads();
    // bitonic sort of the picks, largest key first
    for (int k = 2; k <= P; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            const int o = tid ^ j;
            if (tid < P && o > tid) {
                const unsigned long long ka = s.key[tid], kb = s.key[o];
                if (((tid & k) == 0) ? ka < kb : ka > kb) { s.key[tid] = kb; s.key[o] = ka; }
            }
            __syncthreads();
        }
    }
    return npick;
}

__global__ void __launch_bounds__(BEAM_WIDE_THREADS) beam_wide_select_kernel(BeamWideArgs w) {
    pdl_wait();
    __shared__ BeamRadixSmem s;
    const BeamSelectArgs& a = w.s;
    const int b = blockIdx.x, tid = threadIdx.x;
    const int n = a.K * a.KK;
    const int npick = beam_radix_topk(w.mono + (size_t)b * n, n, a.K, s);
    if (tid < a.K) {
        if (tid < npick) {
            const int f = beam_key_flat(s.key[tid]), p = f / a.KK;
            const size_t e = (size_t)b * n + f;
            beam_emit(a, b, tid, p, a.cand_tok[e], a.beam_logps[(size_t)b * a.K + p] + a.cand_logp[e]);
        } else {
            beam_fill(a, b, tid);
        }
    }
}

}  // namespace grb
