// genrec_b200 - shared device helpers (sm_90a).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <mutex>
#include <utility>

namespace grb {

typedef __nv_bfloat16 bf16;

#define GRB_DEVINL __device__ __forceinline__

// ----------------------------------------------------------------------------- programmatic dependent launch
// Every kernel starts with pdl_wait() (before any global access and before any early exit): when launched with the
// programmatic-stream-serialization attribute its CTAs may be scheduled while the previous kernel on the stream drains,
// and this instruction is where they stop until that kernel has completed and its writes are visible.  It is a no-op
// for an ordinary launch.  Right after it the CTA releases ITS dependents: the release fires once every CTA of this grid
// has started (and therefore passed its own wait), so the next kernel's CTAs fill SMs as this grid's last wave drains
// and never compete with CTAs of this grid that are still to be scheduled; look-ahead is exactly one kernel.  Data
// ordering stays the stream's own (each dependent waits for full completion of this grid) - only launch latency and
// the per-CTA prologue (barrier init, descriptor prefetch) move off the critical path.
GRB_DEVINL void pdl_wait() {
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

inline bool pdl_enabled() {
    static int v = -1;
    if (v < 0) {
        const char* e = getenv("GRB_PDL");
        v = (e && e[0] == '0') ? 0 : 1;
    }
    return v != 0;
}

// opt in to > 48 KB dynamic shared memory once per (kernel, high-water mark): no runtime call on the steady-state path,
// in particular none while a CUDA graph is being captured after warm-up.
template <class Kern>
inline cudaError_t set_max_smem(Kern k, size_t bytes) {
    static std::mutex mu;
    // keyed by (device, kernel address): the attribute is per device.  One map per instantiation, that is per kernel signature.
    static std::map<std::pair<int, const void*>, size_t> high_water;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lock(mu);
    size_t& hw = high_water[std::make_pair(dev, reinterpret_cast<const void*>(k))];
    if (hw < 48 * 1024) hw = 48 * 1024;
    if (bytes > hw) {
        cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
        if (e != cudaSuccess) return e;
        hw = bytes;
    }
    return cudaSuccess;
}

// Every kernel launch of the library goes through launch_kc, which also counts them (grb_launch_count in the C ABI).
inline unsigned long long& launch_counter() {
    static unsigned long long n = 0;
    return n;
}
// launch_kc(kernel, grid, block, cluster, smem, st, args...) with the PDL attribute (GRB_PDL=0 turns it off) and, for cluster > 1, a
// thread-block cluster of `cluster` CTAs along x; launch_k is the same without clusters.  A launch with more than 48 KB of dynamic
// shared memory first raises the kernel's limit through set_max_smem.  The result is this launch's own error: the opt-in's, or
// cudaLaunchKernelEx's, never one an earlier runtime call left behind.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_kc(void (*kern)(KArgs...), dim3 grid, dim3 block, unsigned cluster, size_t smem, cudaStream_t st, Args&&... args) {
    if (smem > 48 * 1024) {
        const cudaError_t e = set_max_smem(kern, smem);
        if (e != cudaSuccess) return e;
    }
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute at[2];
    unsigned n = 0;
    if (pdl_enabled()) {
        at[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[n].val.programmaticStreamSerializationAllowed = 1;
        ++n;
    }
    if (cluster > 1) {
        at[n].id = cudaLaunchAttributeClusterDimension;
        at[n].val.clusterDim.x = cluster;
        at[n].val.clusterDim.y = 1;
        at[n].val.clusterDim.z = 1;
        ++n;
    }
    cfg.attrs = at;
    cfg.numAttrs = n;
    ++launch_counter();
    return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
    return launch_kc(kern, grid, block, 1u, smem, st, static_cast<Args&&>(args)...);
}

// ----------------------------------------------------------------------------- small math
GRB_DEVINL float rcp_fast(float x) {
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
constexpr float kLog2e = 1.4426950408889634f;
GRB_DEVINL float ex2_fast(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
GRB_DEVINL float sigmoidf_fast(float x) { return rcp_fast(1.f + __expf(-x)); }
GRB_DEVINL float siluf(float x) { return x * sigmoidf_fast(x); }
// d/dx silu(x) = s * (1 + x * (1 - s))
GRB_DEVINL float dsiluf(float x) {
    float s = sigmoidf_fast(x);
    return s * (1.f + x * (1.f - s));
}

GRB_DEVINL uint32_t pack_bf16(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}
GRB_DEVINL float2 unpack_bf16(uint32_t u) {
    __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
    return __bfloat1622float2(v);
}
GRB_DEVINL float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

GRB_DEVINL float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
GRB_DEVINL float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// ----------------------------------------------------------------------------- packed (jagged) batches
// First row and length of sequence b.  A malformed device `offsets` yields wrong numbers but never a row outside [0, T).
// The attention and embedding kernels take JAGGED as a template parameter, so that their padded instantiations keep
// the registers (and the code) they had before packed batches existed.
template <bool JAGGED = true>
GRB_DEVINL void seq_span(const long long* offsets, int T, int L, int b, long long& tok0, int& len) {
    if (!JAGGED || offsets == nullptr) {
        tok0 = (long long)b * L;
        len = L;
        return;
    }
    long long lo = offsets[b], hi = offsets[b + 1];
    lo = lo < 0 ? 0 : (lo > T ? T : lo);
    hi = hi < lo ? lo : (hi > T ? T : hi);
    tok0 = lo;
    len = (int)(hi - lo < L ? hi - lo : L);
}

// ----------------------------------------------------------------------------- dropout RNG
// Counter-based: keep(seed, site, row, col) is a pure function, so the backward pass re-derives the forward mask
// instead of storing it.  Elements are addressed by (row, column) of the [rows, cols] operand the mask belongs to -
// 32-bit arithmetic only.  A row contributes two mixed keys (computed once per row and thread); one two-round
// multiply / xor-shift mix per column PAIR then serves two neighbouring columns: column c takes the low (c even) or
// high (c odd) 16 bits of the pair's hash and is dropped when they are below a 16-bit threshold (p is honoured to
// 2^-16 and the keep scale is the exact reciprocal of the realised keep probability, so the expectation is
// unchanged).  tests/test_linear_gpu.py restates the function in numpy and checks masks bit for bit, plus the
// row/column cross-correlations against those of an ideal generator.
struct DropRowKeys {
    uint32_t ka, kb;
};
struct Dropout {
    uint64_t seed;
    const unsigned long long* seed_dev;  // nullable: *seed_dev is added to seed at kernel start (CUDA-graph-safe reseeding)
    uint32_t thresh;  // drop when the element's 16 random bits < thresh ; thresh = round(p * 2^16)
    float scale;      // 2^16 / (2^16 - thresh) ; p == 0 -> thresh = 0, scale = 1
    uint32_t site;
    GRB_DEVINL void resolve() {
        if (thresh != 0u && seed_dev) seed += *seed_dev;
        seed_dev = nullptr;
    }
    GRB_DEVINL DropRowKeys row_keys(uint32_t row) const {
        const uint32_t k0 = (uint32_t)seed ^ (site * 0x9E3779B1u), k1 = (uint32_t)(seed >> 32) + 0x7F4A7C15u;
        DropRowKeys r;
        r.ka = (row ^ k1) * 0x9E3779B1u;
        r.ka ^= r.ka >> 16;
        uint32_t b = r.ka * 0x846CA68Bu;
        b ^= b >> 15;
        r.kb = k0 ^ b;
        return r;
    }
    static GRB_DEVINL uint32_t pair_hash(const DropRowKeys& r, uint32_t colpair) {
        uint32_t x = (colpair ^ r.kb) * 0x7FEB352Du;
        x ^= x >> 15;
        x ^= r.ka;
        x *= 0x846CA68Bu;
        x ^= x >> 16;
        return x;
    }
    GRB_DEVINL float apply(float v, uint32_t row, uint32_t col) const {
        if (thresh == 0u) return v;
        const uint32_t h = pair_hash(row_keys(row), col >> 1);
        const uint32_t u = (col & 1u) ? (h >> 16) : (h & 0xffffu);
        return u < thresh ? 0.f : v * scale;
    }
    // two neighbouring columns 2 * colpair, 2 * colpair + 1 with one hash
    GRB_DEVINL void apply2p(float& v0, float& v1, uint32_t row, uint32_t colpair) const {
        if (thresh == 0u) return;
        const uint32_t h = pair_hash(row_keys(row), colpair);
        v0 = (h & 0xffffu) < thresh ? 0.f : v0 * scale;
        v1 = (h >> 16) < thresh ? 0.f : v1 * scale;
    }
    GRB_DEVINL void apply2(float& v0, float& v1, uint32_t row, uint32_t col_even) const { apply2p(v0, v1, row, col_even >> 1); }
};
inline Dropout make_dropout(float p, uint64_t seed, uint32_t site, const void* seed_dev = nullptr) {
    Dropout d;
    d.seed = seed;
    d.seed_dev = static_cast<const unsigned long long*>(seed_dev);
    d.site = site;
    double t = (double)p * 65536.0 + 0.5;
    d.thresh = p <= 0.f ? 0u : (t >= 65536.0 ? 65536u : (uint32_t)t);
    d.scale = d.thresh >= 65536u ? 0.f : 65536.f / (float)(65536u - d.thresh);
    return d;
}

// ----------------------------------------------------------------------------- async copy / ldmatrix / mma.sync
GRB_DEVINL uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// 16-byte global->shared async copy; src_bytes == 0 zero-fills the destination.
GRB_DEVINL void cp_async16(void* smem_dst, const void* gmem_src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_u32(smem_dst)), "l"(gmem_src),
                 "r"(src_bytes));
}
// 16-byte vector reduction into global fp32 (address 16-byte aligned): one L2 atomic transaction for four elements
GRB_DEVINL void red_add_v4(float* addr, float a, float b, float c, float d) {
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
GRB_DEVINL void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
GRB_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
GRB_DEVINL void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

GRB_DEVINL void ldsm_x4(uint32_t (&r)[4], const void* smem_row_ptr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_u32(smem_row_ptr)));
}
GRB_DEVINL void ldsm_x4_t(uint32_t (&r)[4], const void* smem_row_ptr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(smem_u32(smem_row_ptr)));
}

// D(16x8,f32) += A(16x16,bf16,row) * B(16x8,bf16,col)
GRB_DEVINL void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// d = a * b (no accumulator input: the zero C operand becomes RZ, so callers need not clear d first)
GRB_DEVINL void mma_bf16_z(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%10,%10,%10,%10};\n"
        : "=f"(d[0]), "=f"(d[1]), "=f"(d[2]), "=f"(d[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1), "f"(0.f));
}

// Fragment address helpers (lane -> row/col of the 8x8 matrix row this lane points at), see the PTX ISA, mma.m16n8k16 fragment layouts.
// A operand, smem tile stored [m][k] (k contiguous): non-transposed ldmatrix.
GRB_DEVINL int lane_a_row(int lane) { return (lane & 7) + ((lane >> 3) & 1) * 8; }
GRB_DEVINL int lane_a_col(int lane) { return (lane >> 4) * 8; }
// B operand, smem tile stored [n][k] (k contiguous): non-transposed ldmatrix, two n-tiles per x4.
GRB_DEVINL int lane_b_row(int lane) { return (lane & 7) + (lane >> 4) * 8; }
GRB_DEVINL int lane_b_col(int lane) { return ((lane >> 3) & 1) * 8; }
// B operand, smem tile stored [k][n] (n contiguous): transposed ldmatrix, two n-tiles per x4  (== lane_a_row/col).
// A operand, smem tile stored [k][m] (m contiguous): transposed ldmatrix                      (== lane_b_row/col with row=k, col=m).


// ----------------------------------------------------------------------------- deterministic cross-CTA sums
// Float atomics from many CTAs add in whatever order the CTAs finish, so the last bits of a gradient (and through Adam the
// parameters) would change from run to run.  The cross-CTA reductions of the training step are split in two instead: each CTA
// stores its partials to scratch from the caller's workspace (det_store, layout [group][member][W]), and det_finish_kernel,
// launched right after on the same stream, sums them in a fixed order and adds the result once.
template <class F>
GRB_DEVINL void det_store(float* part, int group, int member, int nmembers, int W, int n, F vals) {
    float* dst = part + ((size_t)group * nmembers + member) * W;
    for (int i = threadIdx.x; i < n; i += blockDim.x) dst[i] = vals(i);
}
struct DetFinishArgs {
    const float* part;
    int ngroups, nmembers, W;
    int gpo, gstride, estride;   // group g, element i -> out[g / gpo][(g % gpo) * gstride + i * estride], kept when that index < len
    float* out[4];
    int len[4];
};
// one warp per (group, element): lane l sums members l, l + 32, ... in order, then a fixed butterfly
__global__ void __launch_bounds__(256) det_finish_kernel(DetFinishArgs a) {
    pdl_wait();
    const int w = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    const int g = w / a.W, i = w % a.W;
    if (g >= a.ngroups) return;
    const int k = g / a.gpo, idx = (g % a.gpo) * a.gstride + i * a.estride;
    if (idx >= a.len[k]) return;
    const float* p = a.part + (size_t)g * a.nmembers * a.W + i;
    float s = 0.f;
#pragma unroll 4
    for (int m = lane; m < a.nmembers; m += 32) s += p[(size_t)m * a.W];
    s = warp_sum(s);
    if (lane == 0) atomicAdd(a.out[k] + idx, s);   // one add per element and launch
}

}  // namespace grb
